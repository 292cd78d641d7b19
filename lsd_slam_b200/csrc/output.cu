// output.cu -- what leaves the device, through the C ABI (include/lsdgpu.h): one keyframe packed as keyframeMsg.pointcloud
// (output.cuh), and the resident map exported as one filtered world-frame point cloud (cloud.cuh).
#include "internal.cuh"
#include "output.cuh"
#include "cloud.cuh"

#include <algorithm>
#include <cmath>

// ------------------------------------------------------------------------------------------------------
// keyframe output formats (SURVEY 8f row 4)
// ------------------------------------------------------------------------------------------------------
// The request of lsdgpu_keyframe_pack_pointcloud and its device twin: checks the keyframe and level, returns the record count
static int packRequest(lsdgpu_ctx* ctx, int kf_id, int publish_level, FrameSlot** slot, int* n)
{
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return failMissing(ctx, kf_id, "unknown keyframe id");
    if (publish_level < 0 || publish_level >= LSD_LEVELS) return lsd_fail(ctx, "bad level");
    if (!kf->hasDepth) return lsd_fail(ctx, "keyframe has no depth");
    *slot = kf;
    *n = (ctx->w >> publish_level) * (ctx->h >> publish_level);
    return 0;
}
// the packing kernel of an accepted request, writing into `out` (the staging buffer or a caller's)
static int packPointcloud(lsdgpu_ctx* ctx, FrameSlot* kf, int publish_level, int n, uint32_t* out)
{
    int r = ensureIdepthPyramid(ctx, kf);                      // f->idepth(publishLvl), ROSOutput3DWrapper.cpp:96-97
    if (r) return r;
    k_pack_pointcloud<<<divUp(3 * n, 256), 256, 0, ctx->stream>>>(kf->idepth[publish_level], kf->idepthVar[publish_level],
                                                                  kf->image[publish_level], n, out);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    return 0;
}

extern "C" int lsdgpu_keyframe_pack_pointcloud(lsdgpu_ctx* ctx, int kf_id, int publish_level, lsdgpu_input_point_dense* out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf;
    int n;
    int r = packRequest(ctx, kf_id, publish_level, &kf, &n);
    if (r || (r = packPointcloud(ctx, kf, publish_level, n, ctx->dPacked))) return r;
    LSD_CHECK(ctx, cudaMemcpyAsync(out, ctx->dPacked, (size_t)n * 12, cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int lsdgpu_keyframe_pack_pointcloud_device(lsdgpu_ctx* ctx, int kf_id, int publish_level, lsdgpu_input_point_dense* d_out,
                                                      size_t capacity, void* stream)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf;
    int n;
    int r = packRequest(ctx, kf_id, publish_level, &kf, &n);
    if (r || (r = checkCapacity(ctx, "keyframe_pack_pointcloud_device", "the point cloud", (size_t)n * 12, capacity))) return r;
    if ((r = checkDevicePtr(ctx, "keyframe_pack_pointcloud_device", "the output", d_out, 4))) return r;
    LSD_CHECK(ctx, afterCallerStream(ctx, stream));
    if ((r = packPointcloud(ctx, kf, publish_level, n, (uint32_t*)d_out))) return r;
    LSD_CHECK(ctx, beforeCallerStream(ctx, stream));
    return 0;
}

// ------------------------------------------------------------------------------------------------------
// the resident map as one point cloud: lsd_slam_viewer's KeyFrameDisplay::refreshPC + flushPC (cloud.cuh)
// ------------------------------------------------------------------------------------------------------
extern "C" void lsdgpu_default_cloud_filter(lsdgpu_cloud_filter* f)
{   // lsd_slam_viewer/src/settings.cpp:36-40
    f->scaledDepthVarTH = 1; f->absDepthVarTH = 1; f->minNearSupport = 5; f->sparsifyFactor = 1;
}

static void cloudShape(const lsdgpu_ctx* ctx, int level, int* rows, int* tilesPerKf)
{
    const int w = ctx->w >> level, h = ctx->h >> level;
    *rows = std::max(1, CLOUD_TILE_PX / w);
    *tilesPerKf = divUp(h - 2, *rows);
}

// ticket + 2 counts per keyframe, then the tile states
static size_t cloudHeaderBytes(int maxKf) { return alignUp(16 + (size_t)maxKf * 8, 256); }

void cloudRelease(lsdgpu_ctx* ctx)
{
    if (ctx->cloudCopyStream) {
        cudaStreamSynchronize(ctx->cloudCopyStream);
        cudaStreamDestroy(ctx->cloudCopyStream);
        for (int i = 0; i < 2; i++) { cudaEventDestroy(ctx->cloudKernDone[i]); cudaEventDestroy(ctx->cloudCopyDone[i]); }
        cudaEventDestroy(ctx->cloudT0); cudaEventDestroy(ctx->cloudT1);
    }
    if (ctx->cloudMem) cudaFree(ctx->cloudMem);
    if (ctx->hCloudMem) cudaFreeHost(ctx->hCloudMem);
    ctx->cloudCopyStream = nullptr; ctx->cloudT0 = ctx->cloudT1 = nullptr;
    ctx->cloudMem = ctx->hCloudMem = nullptr;
    ctx->cloudMaxKf = 0; ctx->cloudTimed = false;
}

// What every export needs of the kernel for the context's frame size: a frame narrow enough for it, and its dynamic shared-memory
// limit raised where a level stages more than 48 KB.  -> the largest number of tiles of one keyframe over the levels
static int cloudKernelSetup(lsdgpu_ctx* ctx, const char* fn, int* maxTilesOut)
{
    if (ctx->w - 2 > CLOUD_MAX_ITERS * CLOUD_THREADS) {
        char msg[160];
        snprintf(msg, sizeof(msg), "%s: frame too wide for the export kernel", fn);
        return lsd_fail(ctx, msg);
    }
    int maxTiles = 0;
    size_t maxSmem = 0;
    for (int l = 0; l < LSD_LEVELS && (ctx->w >> l) >= 3 && (ctx->h >> l) >= 3; l++) {
        int rows, tiles;
        cloudShape(ctx, l, &rows, &tiles);
        maxTiles = std::max(maxTiles, tiles);
        maxSmem = std::max(maxSmem, (size_t)(rows + 2) * (ctx->w >> l) * 4);
    }
    if (maxSmem > 48 * 1024)
        LSD_CHECK(ctx, cudaFuncSetAttribute(k_cloud_export, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)maxSmem));
    *maxTilesOut = maxTiles;
    return 0;
}

// (float)(c / 255.0) for c = 0..255: KeyFrameDisplay.cpp:331, uchar / double, rounded to float
static void cloudIntensityTable(float* tab)
{
    for (int c = 0; c < 256; c++) tab[c] = (float)(c / 255.0);
}

extern "C" int lsdgpu_cloud_reserve(lsdgpu_ctx* ctx, int maxKf)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (maxKf <= 0) return lsd_fail(ctx, "cloud_reserve: max_keyframes_per_launch must be positive");
    int maxTiles;
    int r = cloudKernelSetup(ctx, "cloud_reserve", &maxTiles);
    if (r) return r;
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    cloudRelease(ctx);
    const size_t kfBytes = alignUp((size_t)maxKf * sizeof(CloudKf), 256);
    ctx->cloudStateBytes = cloudHeaderBytes(maxKf) + alignUp((size_t)maxKf * maxTiles * 8, 256);
    const size_t outBytes = alignUp((size_t)maxKf * (ctx->w - 2) * (ctx->h - 2) * 16, 256);
    const size_t cntBytes = alignUp((size_t)maxKf * 8, 256);
    LSD_CHECK(ctx, cudaMalloc((void**)&ctx->cloudMem, 2 * (kfBytes + ctx->cloudStateBytes + outBytes) + 1024));
    LSD_CHECK(ctx, cudaHostAlloc((void**)&ctx->hCloudMem, 2 * (kfBytes + cntBytes), cudaHostAllocDefault));
    char* p = ctx->cloudMem;
    char* hp = ctx->hCloudMem;
    for (int i = 0; i < 2; i++) {
        ctx->dCloudKfs[i] = p; p += kfBytes;
        ctx->dCloudState[i] = (unsigned long long*)p; p += ctx->cloudStateBytes;
        ctx->dCloudOut[i] = (float4*)p; p += outBytes;
        ctx->hCloudKfs[i] = hp; hp += kfBytes;
        ctx->hCloudCounts[i] = (int*)hp; hp += cntBytes;
    }
    ctx->dCloudIntensity = (float*)p;
    float tab[256];
    cloudIntensityTable(tab);
    LSD_CHECK(ctx, cudaMemcpy(ctx->dCloudIntensity, tab, sizeof(tab), cudaMemcpyHostToDevice));
    LSD_CHECK(ctx, cudaStreamCreateWithFlags(&ctx->cloudCopyStream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; i++) {
        LSD_CHECK(ctx, cudaEventCreateWithFlags(&ctx->cloudKernDone[i], cudaEventDisableTiming));
        LSD_CHECK(ctx, cudaEventCreateWithFlags(&ctx->cloudCopyDone[i], cudaEventDisableTiming));
        LSD_CHECK(ctx, cudaEventRecord(ctx->cloudKernDone[i], ctx->stream));
        LSD_CHECK(ctx, cudaEventRecord(ctx->cloudCopyDone[i], ctx->cloudCopyStream));
    }
    LSD_CHECK(ctx, cudaEventCreate(&ctx->cloudT0));
    LSD_CHECK(ctx, cudaEventCreate(&ctx->cloudT1));
    ctx->cloudMaxKf = maxKf;
    return 0;
}

// The arguments both exports check, in the host export's order; the reservation is checked by `reserved` (the host export) only.
// -> the filter in force and the keyframes' frames
static int cloudRequest(lsdgpu_ctx* ctx, int n, const int* kf_ids, const float* camToWorld, int level, const lsdgpu_cloud_filter* f,
                        int layout, bool reserved, lsdgpu_cloud_filter& flt, std::vector<FrameSlot*>& kfs)
{
    char msg[256];
    if (f) flt = *f;
    else lsdgpu_default_cloud_filter(&flt);
    if (n < 0 || (n > 0 && (!kf_ids || !camToWorld))) return lsd_fail(ctx, "map_export_pointcloud: bad keyframe list");
    if (level < 0 || level >= LSD_LEVELS || (ctx->w >> level) < 3 || (ctx->h >> level) < 3) {
        snprintf(msg, sizeof(msg), "map_export_pointcloud: bad level %d", level);
        return lsd_fail(ctx, msg);
    }
    if (layout != LSDGPU_CLOUD_PLY && layout != LSDGPU_CLOUD_VERTEX) {
        snprintf(msg, sizeof(msg), "map_export_pointcloud: bad layout %d", layout);
        return lsd_fail(ctx, msg);
    }
    if (flt.sparsifyFactor != 1) {
        snprintf(msg, sizeof(msg), "map_export_pointcloud: sparsifyFactor %d is not supported (only 1: the viewer draws rand())",
                 flt.sparsifyFactor);
        return lsd_fail(ctx, msg);
    }
    if (reserved && ctx->cloudMaxKf == 0) return lsd_fail(ctx, "map_export_pointcloud: no reservation (call lsdgpu_cloud_reserve first)");
    kfs.assign(n, nullptr);
    for (int i = 0; i < n; i++) {
        kfs[i] = level == 0 ? findFrame(ctx, kf_ids[i]) : findSlot(ctx, kf_ids[i]);   // level 0 of a minimized keyframe: its record
        if (!kfs[i] && level > 0 && findMinimized(ctx, kf_ids[i])) {
            snprintf(msg, sizeof(msg), "map_export_pointcloud: keyframe %d (kf_ids[%d]) is minimized: only level 0 is kept", kf_ids[i], i);
            return lsd_fail(ctx, msg);
        }
        if (!kfs[i] || !kfs[i]->hasDepth) {
            snprintf(msg, sizeof(msg), "map_export_pointcloud: keyframe %d (kf_ids[%d]) %s", kf_ids[i], i,
                     kfs[i] ? "has no depth" : "is unknown");
            return lsd_fail(ctx, msg);
        }
    }
    return 0;
}

// one keyframe's descriptor (a = its 7 camToWorld floats): the Sim3f of keyframeMsg.camToWorld (KeyFrameDisplay.cpp:68) and its scale (:143),
// rxso3.hpp:263-269; the norm is Eigen's redux tree over the 4 coefficients: (x^2 + y^2) + (z^2 + w^2)
static void cloudDescriptor(const LevelCam& cam, const float* a, const FrameSlot* s_, int level, CloudKf& d)
{
    const float s = std::sqrt((a[0] * a[0] + a[1] * a[1]) + (a[2] * a[2] + a[3] * a[3]));
    for (int k = 0; k < 4; k++) d.nq[k] = a[k] / s;
    d.scale = s;
    d.t[0] = a[4]; d.t[1] = a[5]; d.t[2] = a[6];
    d.fxi = 1 / cam.fx; d.fyi = 1 / cam.fy;             // KeyFrameDisplay::setFrom, :75-78
    d.cxi = -cam.cx / cam.fx; d.cyi = -cam.cy / cam.fy;
    d.idepth = s_->idepth[level]; d.idepthVar = s_->idepthVar[level]; d.image = s_->image[level];
}

// Frame::idepth(level) of every keyframe, as lsdgpu_keyframe_pack_pointcloud
static int cloudPyramids(lsdgpu_ctx* ctx, int level, const std::vector<FrameSlot*>& kfs)
{
    if (level > 0)
        for (FrameSlot* s : kfs) {
            const int r = ensureIdepthPyramid(ctx, s);
            if (r) return r;
        }
    return 0;
}

extern "C" int lsdgpu_map_export_pointcloud(lsdgpu_ctx* ctx, int n, const int* kf_ids, const float* camToWorld, int level,
                                            const lsdgpu_cloud_filter* f, int layout, void* out, int64_t capacity,
                                            int64_t* n_points_out, int32_t* counts)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    char msg[256];
    lsdgpu_cloud_filter flt;
    std::vector<FrameSlot*> kfs;
    int r = cloudRequest(ctx, n, kf_ids, camToWorld, level, f, layout, true, flt, kfs);
    if (r || (r = cloudPyramids(ctx, level, kfs))) return r;
    const LevelCam& cam = ctx->cam[level];
    const int w = cam.w, h = cam.h, maxKf = ctx->cloudMaxKf, nBatches = divUp(n, maxKf);
    int rows, tilesPerKf;
    cloudShape(ctx, level, &rows, &tilesPerKf);
    const size_t smem = (size_t)(rows + 2) * w * 4;
    const int64_t bound = (int64_t)n * (w - 2) * (h - 2);
    std::vector<int32_t> cnt((size_t)2 * n, 0);
    ctx->cloudTimed = false;

    auto launchBatch = [&](int b, bool emit) -> int {
        const int set = b & 1, i0 = b * maxKf, nb = std::min(maxKf, n - i0);
        LSD_CHECK(ctx, cudaEventSynchronize(ctx->cloudKernDone[set]));       // batch b-2 has read this set's descriptors
        CloudKf* hk = (CloudKf*)ctx->hCloudKfs[set];
        for (int j = 0; j < nb; j++) cloudDescriptor(cam, camToWorld + 7 * (size_t)(i0 + j), kfs[i0 + j], level, hk[j]);
        LSD_CHECK(ctx, cudaMemcpyAsync(ctx->dCloudKfs[set], hk, nb * sizeof(CloudKf), cudaMemcpyHostToDevice, ctx->stream));
        LSD_CHECK(ctx, cudaStreamWaitEvent(ctx->stream, ctx->cloudCopyDone[set], 0));   // batch b-2's points have left the buffer
        char* st = (char*)ctx->dCloudState[set];
        LSD_CHECK(ctx, cudaMemsetAsync(st, 0, cloudHeaderBytes(maxKf) + (size_t)nb * tilesPerKf * 8, ctx->stream));
        CloudParams P;
        P.kfs = (const CloudKf*)ctx->dCloudKfs[set];
        P.w = w; P.h = h; P.rows = rows; P.tilesPerKf = tilesPerKf;
        P.scaledTH = flt.scaledDepthVarTH; P.absTH = flt.absDepthVarTH; P.minNearSupport = flt.minNearSupport;
        P.layout = layout; P.emit = emit ? 1 : 0;
        P.intensity = ctx->dCloudIntensity;
        P.ticket = (unsigned int*)st;
        P.counts = (int*)(st + 16);
        P.tileState = (unsigned long long*)(st + cloudHeaderBytes(maxKf));
        P.out = ctx->dCloudOut[set];
        if (!ctx->cloudTimed) { LSD_CHECK(ctx, cudaEventRecord(ctx->cloudT0, ctx->stream)); ctx->cloudTimed = true; }
        k_cloud_export<<<nb * tilesPerKf, CLOUD_THREADS, smem, ctx->stream>>>(P);
        LAUNCH(ctx);
        LSD_CHECK(ctx, cudaGetLastError());
        LSD_CHECK(ctx, cudaEventRecord(ctx->cloudT1, ctx->stream));
        LSD_CHECK(ctx, cudaMemcpyAsync(ctx->hCloudCounts[set], st + 16, (size_t)nb * 8, cudaMemcpyDeviceToHost, ctx->stream));
        LSD_CHECK(ctx, cudaEventRecord(ctx->cloudKernDone[set], ctx->stream));
        return 0;
    };
    // waits for batch b, takes its counts; returns its number of points
    auto finishBatch = [&](int b, int64_t* kept) -> int {
        const int set = b & 1, i0 = b * maxKf, nb = std::min(maxKf, n - i0);
        LSD_CHECK(ctx, cudaEventSynchronize(ctx->cloudKernDone[set]));
        *kept = 0;
        for (int j = 0; j < nb; j++) {
            cnt[2 * (size_t)(i0 + j)] = ctx->hCloudCounts[set][2 * j];
            cnt[2 * (size_t)(i0 + j) + 1] = ctx->hCloudCounts[set][2 * j + 1];
            *kept += ctx->hCloudCounts[set][2 * j + 1];
        }
        return 0;
    };
    auto report = [&](int64_t total) {
        if (n_points_out) *n_points_out = total;
        if (counts && n) memcpy(counts, cnt.data(), cnt.size() * sizeof(int32_t));
    };

    int64_t total = 0;
    if (!out || capacity < bound) {
        // count pass: the number of points is needed before anything may be written to out
        for (int b = 0; b < nBatches; b++) {
            int64_t kept;
            if ((r = launchBatch(b, false)) || (r = finishBatch(b, &kept))) return r;
            total += kept;
        }
        report(total);
        if (!out) return 0;
        if (total > capacity) {
            snprintf(msg, sizeof(msg), "map_export_pointcloud: %lld points do not fit in %lld", (long long)total, (long long)capacity);
            ctx->err = msg;
            return LSDGPU_CLOUD_ERR_CAPACITY;
        }
    }
    // emit pass: batch b's kernel runs while batch b-1's points are copied out (cloudCopyStream)
    int64_t off = 0;
    for (int b = 0; b <= nBatches; b++) {
        if (b < nBatches && (r = launchBatch(b, true))) return r;
        if (b == 0) continue;
        const int pb = b - 1, set = pb & 1;
        int64_t kept;
        if ((r = finishBatch(pb, &kept))) return r;
        if (off + kept > capacity) return lsd_fail(ctx, "map_export_pointcloud: output overflow");   // unreachable: checked above
        LSD_CHECK(ctx, cudaStreamWaitEvent(ctx->cloudCopyStream, ctx->cloudKernDone[set], 0));
        if (kept)
            LSD_CHECK(ctx, cudaMemcpyAsync((char*)out + off * 16, ctx->dCloudOut[set], (size_t)kept * 16, cudaMemcpyDeviceToHost,
                                           ctx->cloudCopyStream));
        LSD_CHECK(ctx, cudaEventRecord(ctx->cloudCopyDone[set], ctx->cloudCopyStream));
        off += kept;
    }
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->cloudCopyStream));
    report(off);
    return 0;
}

extern "C" int lsdgpu_map_export_pointcloud_device(lsdgpu_ctx* ctx, int n, const int* kf_ids, const float* camToWorld, int level,
                                                   const lsdgpu_cloud_filter* f, int layout, void* d_out, int64_t capacity,
                                                   int64_t* n_points_out, int32_t* counts, void* stream)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    char msg[256];
    lsdgpu_cloud_filter flt;
    std::vector<FrameSlot*> kfs;
    int maxTiles;
    int r = cloudRequest(ctx, n, kf_ids, camToWorld, level, f, layout, false, flt, kfs);
    if (r || (r = cloudKernelSetup(ctx, "map_export_pointcloud_device", &maxTiles))) return r;
    if (d_out && (r = checkDevicePtr(ctx, "map_export_pointcloud_device", "the output", d_out, 16))) return r;
    const LevelCam& cam = ctx->cam[level];
    const int w = cam.w, h = cam.h;
    int rows, tilesPerKf;
    cloudShape(ctx, level, &rows, &tilesPerKf);
    if ((int64_t)n * tilesPerKf > INT32_MAX) {
        snprintf(msg, sizeof(msg), "map_export_pointcloud_device: %d keyframes exceed one launch", n);
        return lsd_fail(ctx, msg);
    }
    if (n == 0) {                                       // nothing to export, nothing to order
        if (n_points_out) *n_points_out = 0;
        return 0;
    }
    if ((r = cloudPyramids(ctx, level, kfs))) return r;
    const size_t smem = (size_t)(rows + 2) * w * 4;
    const int64_t bound = (int64_t)n * (w - 2) * (h - 2);

    // one stream-ordered block: the keyframe descriptors and the intensity table (one upload), then the ticket, the counts and
    // the tile states of all n keyframes
    const size_t kfBytes = alignUp((size_t)n * sizeof(CloudKf), 256), tabBytes = 256 * sizeof(float);
    const size_t stateBytes = cloudHeaderBytes(n) + (size_t)n * tilesPerKf * 8;
    std::vector<char> staged(kfBytes + tabBytes);      // read by the upload below; lives until the call has synchronised
    for (int i = 0; i < n; i++) cloudDescriptor(cam, camToWorld + 7 * (size_t)i, kfs[i], level, ((CloudKf*)staged.data())[i]);
    cloudIntensityTable((float*)(staged.data() + kfBytes));
    std::vector<int32_t> cnt((size_t)2 * n);
    LSD_CHECK(ctx, ensureRecordPool(ctx));
    LSD_CHECK(ctx, afterCallerStream(ctx, stream));
    char* blk = nullptr;
    LSD_CHECK(ctx, cudaMallocFromPoolAsync((void**)&blk, kfBytes + tabBytes + stateBytes, ctx->pool[TIER_DEVICE], ctx->stream));
    char* st = blk + kfBytes + tabBytes;
    CloudParams P;
    P.kfs = (const CloudKf*)blk;
    P.w = w; P.h = h; P.rows = rows; P.tilesPerKf = tilesPerKf;
    P.scaledTH = flt.scaledDepthVarTH; P.absTH = flt.absDepthVarTH; P.minNearSupport = flt.minNearSupport;
    P.layout = layout;
    P.intensity = (const float*)(blk + kfBytes);
    P.ticket = (unsigned int*)st;
    P.counts = (int*)(st + 16);
    P.tileState = (unsigned long long*)(st + cloudHeaderBytes(n));
    P.out = (float4*)d_out;
    // one launch over all n keyframes (emit: the points into d_out), then its counts to the host
    auto launch = [&](bool emit) -> int {
        P.emit = emit ? 1 : 0;
        LSD_CHECK(ctx, cudaMemsetAsync(st, 0, stateBytes, ctx->stream));
        k_cloud_export<<<n * tilesPerKf, CLOUD_THREADS, smem, ctx->stream>>>(P);
        LAUNCH(ctx);
        LSD_CHECK(ctx, cudaGetLastError());
        LSD_CHECK(ctx, cudaMemcpyAsync(cnt.data(), st + 16, cnt.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
        return 0;
    };
    // after the last launch: the block goes back to the pool, the caller's stream waits, the host waits for the counts
    auto finish = [&]() -> int64_t {
        cudaFreeAsync(blk, ctx->stream);
        const cudaError_t e = beforeCallerStream(ctx, stream);
        const cudaError_t e2 = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess || e2 != cudaSuccess) {
            snprintf(msg, sizeof(msg), "map_export_pointcloud_device: %s", cudaGetErrorString(e != cudaSuccess ? e : e2));
            ctx->err = msg;
            return -1;
        }
        int64_t total = 0;
        for (int i = 0; i < n; i++) total += cnt[2 * (size_t)i + 1];
        if (n_points_out) *n_points_out = total;
        if (counts) memcpy(counts, cnt.data(), cnt.size() * sizeof(int32_t));
        return total;
    };
    LSD_CHECK(ctx, cudaMemcpyAsync(blk, staged.data(), kfBytes + tabBytes, cudaMemcpyHostToDevice, ctx->stream));
    if (!d_out || capacity < bound) {
        // count launch: the number of points is needed before anything may be written to d_out
        if ((r = launch(false))) return r;
        if (!d_out) return finish() < 0 ? -1 : 0;
        LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
        int64_t total = 0;
        for (int i = 0; i < n; i++) total += cnt[2 * (size_t)i + 1];
        if (total > capacity) {
            if (finish() < 0) return -1;
            snprintf(msg, sizeof(msg), "map_export_pointcloud_device: %lld points do not fit in %lld", (long long)total, (long long)capacity);
            ctx->err = msg;
            return LSDGPU_CLOUD_ERR_CAPACITY;
        }
    }
    if ((r = launch(true))) return r;
    return finish() < 0 ? -1 : 0;
}

extern "C" int lsdgpu_cloud_last_kernel_ms(lsdgpu_ctx* ctx, float* ms)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (!ctx->cloudTimed) return lsd_fail(ctx, "cloud_last_kernel_ms: no export has run");
    LSD_CHECK(ctx, cudaEventSynchronize(ctx->cloudT1));
    LSD_CHECK(ctx, cudaEventElapsedTime(ms, ctx->cloudT0, ctx->cloudT1));
    return 0;
}
