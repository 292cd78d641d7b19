// frames.cu -- frame slots of the C ABI (include/lsdgpu.h): upload, the device prefetch ring, download, pose / counter setters and
// getters, depth import, the input undistorters in front of the frame construction, and the kernel launches of records.cu.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>

#include "internal.cuh"
#include "frame.cuh"

static FrameSlot* acquireSlot(lsdgpu_ctx* ctx, int id)
{
    FrameSlot* s = findSlot(ctx, id);
    if (s) return s;
    if (findMinimized(ctx, id)) return nullptr;      // a minimized frame keeps its id until it is activated or released
    for (auto& c : ctx->slots)
        if (!c.used) {
            FrameSlot fresh = c;          // keep the pointers
            fresh.id = id; fresh.used = true;
            fresh.hasDepth = fresh.idepthPyrValid = fresh.hasGoodMask = false;
            fresh.depthHasBeenUpdatedFlag = false;
            fresh.meanIdepth = 1.f; fresh.numPoints = 0; fresh.statsPending = false;
            memset(fresh.thisToParent, 0, sizeof(fresh.thisToParent));
            fresh.thisToParent[3] = 1; fresh.thisToParent[7] = 1;
            fresh.parentId = -1; fresh.initialTrackedResidual = 0;
            fresh.numFramesTrackedOnThis = fresh.numMappedOnThis = 0;
            fresh.permaNumPts = 0; fresh.permaSet = false;
            fresh.reactAllocated = false; fresh.reactValid = false;
            c = fresh;
            return &c;
        }
    return nullptr;
}

static int buildFrameFromDeviceU8(lsdgpu_ctx* ctx, FrameSlot* s, const uint8_t* dsrc, int pitch, int src = PYR_U8);

extern "C" int lsdgpu_frame_upload_u8(lsdgpu_ctx* ctx, int frame_id, const uint8_t* gray)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s = acquireSlot(ctx, frame_id);
    if (!s) return failMissing(ctx, frame_id, "no free frame slot (release frames or raise max_frames)");
    const size_t n0 = (size_t)ctx->w * ctx->h;
    // double-buffered staging: only wait for the upload issued two frames ago.  A caller buffer that is already
    // page-locked (cudaHostAlloc / cudaHostRegister, e.g. a camera DMA buffer) is copied from directly -- it must then
    // stay untouched until the frame has been consumed; pageable memory goes through the pinned staging copy.
    const int b = ctx->stageIdx;
    ctx->stageIdx ^= 1;
    LSD_CHECK(ctx, cudaEventSynchronize(ctx->stageDone[b]));
    cudaPointerAttributes pa;
    const bool pinned = cudaPointerGetAttributes(&pa, gray) == cudaSuccess && pa.type == cudaMemoryTypeHost;
    if (!pinned) { cudaGetLastError(); memcpy(ctx->hStage[b], gray, n0); }
    LSD_CHECK(ctx, cudaMemcpyAsync(ctx->dStageU8[b], pinned ? gray : ctx->hStage[b], n0, cudaMemcpyHostToDevice, ctx->stream));
    int r = buildFrameFromDeviceU8(ctx, s, ctx->dStageU8[b], ctx->w);
    LSD_CHECK(ctx, cudaEventRecord(ctx->stageDone[b], ctx->stream));
    return r;
}

extern "C" int lsdgpu_stage_reserve(lsdgpu_ctx* ctx, int n_entries)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (n_entries <= 0) return lsd_fail(ctx, "bad ring size");
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    if (ctx->stageRing) { cudaFree(ctx->stageRing); ctx->stageRing = nullptr; ctx->stageEntries = 0; }
    LSD_CHECK(ctx, cudaMalloc((void**)&ctx->stageRing, (size_t)n_entries * ctx->w * ctx->h));
    ctx->stageEntries = n_entries;
    return 0;
}
extern "C" int lsdgpu_stage_put(lsdgpu_ctx* ctx, int index, const uint8_t* gray)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (index < 0 || index >= ctx->stageEntries) return lsd_fail(ctx, "bad ring index");
    const size_t n0 = (size_t)ctx->w * ctx->h;
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(ctx->hStage[0], gray, n0);
    LSD_CHECK(ctx, cudaMemcpyAsync(ctx->stageRing + (size_t)index * n0, ctx->hStage[0], n0, cudaMemcpyHostToDevice, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}
extern "C" int lsdgpu_frame_from_stage(lsdgpu_ctx* ctx, int frame_id, int index)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (index < 0 || index >= ctx->stageEntries) return lsd_fail(ctx, "bad ring index");
    FrameSlot* s = acquireSlot(ctx, frame_id);
    if (!s) return failMissing(ctx, frame_id, "no free frame slot (release frames or raise max_frames)");
    return buildFrameFromDeviceU8(ctx, s, ctx->stageRing + (size_t)index * ctx->w * ctx->h, ctx->w);
}

extern "C" int lsdgpu_frame_upload_device_u8(lsdgpu_ctx* ctx, int frame_id, const uint8_t* d_gray, size_t pitch, void* stream)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    int r = checkDeviceImage(ctx, "frame_upload_device_u8", d_gray, pitch, ctx->w, ctx->h);
    if (r) return r;
    FrameSlot* s = acquireSlot(ctx, frame_id);
    if (!s) return failMissing(ctx, frame_id, "no free frame slot (release frames or raise max_frames)");
    LSD_CHECK(ctx, afterCallerStream(ctx, stream));
    if ((r = buildFrameFromDeviceU8(ctx, s, d_gray, (int)pitch))) return r;
    LSD_CHECK(ctx, beforeCallerStream(ctx, stream));
    return 0;
}
extern "C" int lsdgpu_stage_put_device(lsdgpu_ctx* ctx, int index, const uint8_t* d_gray, size_t pitch, void* stream)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (index < 0 || index >= ctx->stageEntries) return lsd_fail(ctx, "bad ring index");
    int r = checkDeviceImage(ctx, "stage_put_device", d_gray, pitch, ctx->w, ctx->h);
    if (r) return r;
    LSD_CHECK(ctx, afterCallerStream(ctx, stream));
    LSD_CHECK(ctx, cudaMemcpy2DAsync(ctx->stageRing + (size_t)index * ctx->w * ctx->h, ctx->w, d_gray, pitch, ctx->w, ctx->h,
                                     cudaMemcpyDefault, ctx->stream));
    LSD_CHECK(ctx, beforeCallerStream(ctx, stream));
    return 0;
}

// k_image_pyramid<src> from `dsrc` (`pitch` bytes per row), then k_gradients, over the buffers of slot `s`
static int buildImagePyramid(lsdgpu_ctx* ctx, FrameSlot* s, const uint8_t* dsrc, int pitch, int src)
{
    const int w = ctx->w, h = ctx->h;
    PyrPtrs pp;
    for (int l = 0; l < LSD_LEVELS; l++) pp.l[l] = s->image[l];
    if (src == PYR_PTAM) k_image_pyramid<PYR_PTAM><<<dim3(w / 16, h / 16), 256, 0, ctx->stream>>>(dsrc, pitch, pp, w, h, ctx->dRemapX, ctx->dRemapY, ctx->rawW, nullptr);
    else if (src == PYR_OPENCV)
        k_image_pyramid<PYR_OPENCV><<<dim3(w / 16, h / 16), 256, 0, ctx->stream>>>(dsrc, pitch, pp, w, h, nullptr, nullptr, ctx->rawW,
                                                                                   nullptr, ctx->dCvMap1, ctx->dCvMap2, ctx->rawH);
    else if (src == PYR_F32) k_image_pyramid<PYR_F32><<<dim3(w / 16, h / 16), 256, 0, ctx->stream>>>(dsrc, pitch, pp, w, h);
    else k_image_pyramid<PYR_U8><<<dim3(w / 16, h / 16), 256, 0, ctx->stream>>>(dsrc, pitch, pp, w, h);
    LAUNCH(ctx);
    GradPtrs gp;
    for (int l = 0; l < LSD_LEVELS; l++) { gp.img[l] = s->image[l]; gp.grad[l] = s->grad[l]; gp.w[l] = w >> l; gp.h[l] = h >> l; }
    gp.maxgrad0 = s->maxgrad;
    // blockIdx.y = level; level 0 runs as 32x8 tiles, levels 1..4 linearly (their block counts are smaller than the tile count)
    LSD_CHECK(ctx, launchPDL(k_gradients, dim3(divUp(w, GR_TW) * divUp(h, GR_TH), LSD_LEVELS), dim3(256), 0, ctx->stream, gp));      // + maxGradients of level 0
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    return 0;
}

// dsrc: the u8 image (PYR_U8) or the raw image (PYR_PTAM, PYR_OPENCV), `pitch` bytes per row
static int buildFrameFromDeviceU8(lsdgpu_ctx* ctx, FrameSlot* s, const uint8_t* dsrc, int pitch, int src)
{
    const int r = buildImagePyramid(ctx, s, dsrc, pitch, src);
    if (!r) { s->hasDepth = false; s->idepthPyrValid = false; s->hasGoodMask = false; }
    return r;
}

int buildImagePyramidFromRecord(lsdgpu_ctx* ctx, FrameSlot* s, const float* image0)
{
    return buildImagePyramid(ctx, s, (const uint8_t*)image0, ctx->w * 4, PYR_F32);
}

int launchRecordCopy(lsdgpu_ctx* ctx, const RecordPart* from, const RecordPart* to, int n)
{
    static_assert(REC_PARTS <= REC_MAX_SEGS, "a record's parts are copied in one launch");
    RecordCopy c = {};
    for (int k = 0; k < n; k++) {
        if (!from[k].bytes) continue;
        c.src[c.n] = (const uint4*)*from[k].ptr; c.dst[c.n] = (uint4*)*to[k].ptr;
        c.end[c.n] = (c.n ? c.end[c.n - 1] : 0) + (long long)(alignUp(from[k].bytes, 16) / 16);
        c.n++;
    }
    const long long total = c.end[c.n - 1];
    const int grid = (int)std::min<long long>((total + 255) / 256, (long long)ctx->smCount * 8);
    k_record_copy<<<grid, 256, 0, ctx->stream>>>(c);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    return 0;
}

int ensureIdepthPyramid(lsdgpu_ctx* ctx, FrameSlot* s)
{
    if (!s->hasDepth) return lsd_fail(ctx, "keyframe has no depth");
    if (s->idepthPyrValid) return 0;
    PyrPtrs id, var;
    for (int l = 0; l < LSD_LEVELS; l++) { id.l[l] = s->idepth[l]; var.l[l] = s->idepthVar[l]; }
    k_idepth_pyramid<<<dim3(ctx->w / 16, ctx->h / 16), 256, 0, ctx->stream>>>(id, var, ctx->w, ctx->h);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    s->idepthPyrValid = true;
    return 0;
}

// The plane lsdgpu_frame_download and lsdgpu_frame_download_device copy: checks the request and returns its frame and size
static int downloadPlane(lsdgpu_ctx* ctx, int frame_id, int what, int level, FrameSlot** slot, size_t* bytes)
{
    FrameSlot* s = findFrame(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    if (level < 0 || level >= LSD_LEVELS) return lsd_fail(ctx, "bad level");
    if ((s->record[TIER_DEVICE] || s->record[TIER_HOST]) && !(level == 0 && (what == LSDGPU_BUF_IMAGE || what == LSDGPU_BUF_IDEPTH || what == LSDGPU_BUF_IDEPTH_VAR))) {
        ctx->err = "frame " + std::to_string(frame_id) + " is minimized: only image, idepth and idepthVar of level 0 are kept (lsdgpu_frame_activate it first)";
        return -2;
    }
    const size_t n = ((size_t)ctx->w * ctx->h) >> (2 * level);
    switch (what) {
    case LSDGPU_BUF_IMAGE: *bytes = n * 4; break;
    case LSDGPU_BUF_GRADIENTS: *bytes = n * 16; break;
    case LSDGPU_BUF_MAXGRAD: if (level != 0) return lsd_fail(ctx, "maxGradients exists at level 0 only"); *bytes = n * 4; break;
    case LSDGPU_BUF_IDEPTH:
    case LSDGPU_BUF_IDEPTH_VAR: if (!s->hasDepth) return lsd_fail(ctx, "frame has no depth"); *bytes = n * 4; break;
    case LSDGPU_BUF_GOODMASK: *bytes = ((size_t)ctx->w * ctx->h) / 4; break;
    default: return lsd_fail(ctx, "bad buffer selector");
    }
    *slot = s;
    return 0;
}
// its source, once the request has been accepted: builds the idepth pyramid if needed; nullptr for a good mask that was never
// written (it reads as all 1s, Frame.h:433: initialised to true)
static int downloadSource(lsdgpu_ctx* ctx, FrameSlot* s, int what, int level, const void** src)
{
    switch (what) {
    case LSDGPU_BUF_IMAGE: *src = s->image[level]; break;
    case LSDGPU_BUF_GRADIENTS: *src = s->grad[level]; break;
    case LSDGPU_BUF_MAXGRAD: *src = s->maxgrad; break;
    case LSDGPU_BUF_IDEPTH:
    case LSDGPU_BUF_IDEPTH_VAR:
        if (level > 0) { int r = ensureIdepthPyramid(ctx, s); if (r) return r; }
        *src = (what == LSDGPU_BUF_IDEPTH) ? s->idepth[level] : s->idepthVar[level]; break;
    default: *src = s->hasGoodMask ? s->goodMask : nullptr; break;
    }
    return 0;
}

extern "C" int lsdgpu_frame_download(lsdgpu_ctx* ctx, int frame_id, int what, int level, void* out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s;
    size_t bytes;
    const void* src;
    int r = downloadPlane(ctx, frame_id, what, level, &s, &bytes);
    if (r || (r = downloadSource(ctx, s, what, level, &src))) return r;
    if (!src) { memset(out, 1, bytes); return 0; }
    // from an offloaded frame's host body the copy is host to host, which cudaMemcpyAsync need not order behind the stream
    if (s->record[TIER_HOST]) LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    LSD_CHECK(ctx, cudaMemcpyAsync(out, src, bytes, cudaMemcpyDefault, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int lsdgpu_frame_download_device(lsdgpu_ctx* ctx, int frame_id, int what, int level, void* d_out, size_t capacity, void* stream)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s;
    size_t bytes;
    const void* src;
    int r = downloadPlane(ctx, frame_id, what, level, &s, &bytes);
    if (r || (r = checkCapacity(ctx, "frame_download_device", "the plane", bytes, capacity))) return r;
    if ((r = checkDevicePtr(ctx, "frame_download_device", "the output", d_out,
                            what == LSDGPU_BUF_GRADIENTS ? 16 : what == LSDGPU_BUF_GOODMASK ? 1 : 4)))
        return r;
    LSD_CHECK(ctx, afterCallerStream(ctx, stream));
    if ((r = downloadSource(ctx, s, what, level, &src))) return r;
    if (src) LSD_CHECK(ctx, cudaMemcpyAsync(d_out, src, bytes, cudaMemcpyDefault, ctx->stream));
    else LSD_CHECK(ctx, cudaMemsetAsync(d_out, 1, bytes, ctx->stream));
    LSD_CHECK(ctx, beforeCallerStream(ctx, stream));
    return 0;
}

// Frame::setDepthFromGroundTruth from a device plane of metric depth, `stride` floats per row
static int setDepthGT(lsdgpu_ctx* ctx, FrameSlot* s, const float* ddepth, int stride, float cov_scale)
{
    k_set_depth_gt<<<divUp(ctx->w * ctx->h, 256), 256, 0, ctx->stream>>>(ddepth, stride, s->maxgrad, s->idepth[0], s->idepthVar[0],
                                                                         ctx->w, ctx->h, ctx->g.minUseGrad, cov_scale);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    s->hasDepth = true; s->idepthPyrValid = false;
    return 0;
}

extern "C" int lsdgpu_frame_set_depth_gt(lsdgpu_ctx* ctx, int frame_id, const float* depth, float cov_scale)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return failMissing(ctx, frame_id, "unknown frame id");
    const int n = ctx->w * ctx->h;
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(ctx->hStageF, depth, (size_t)n * 4);
    LSD_CHECK(ctx, cudaMemcpyAsync(ctx->dStageF, ctx->hStageF, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    return setDepthGT(ctx, s, ctx->dStageF, ctx->w, cov_scale);
}

extern "C" int lsdgpu_frame_set_depth_gt_device(lsdgpu_ctx* ctx, int frame_id, const float* d_depth, size_t pitch, float cov_scale,
                                                void* stream)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return failMissing(ctx, frame_id, "unknown frame id");
    int r = checkDevicePlaneF32(ctx, "frame_set_depth_gt_device", "the depth", d_depth, pitch);
    if (r) return r;
    LSD_CHECK(ctx, afterCallerStream(ctx, stream));
    if ((r = setDepthGT(ctx, s, d_depth, (int)(pitch / 4), cov_scale))) return r;
    LSD_CHECK(ctx, beforeCallerStream(ctx, stream));
    return 0;
}

extern "C" int lsdgpu_frame_set_idepth(lsdgpu_ctx* ctx, int frame_id, const float* idepth, const float* idepthVar)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return failMissing(ctx, frame_id, "unknown frame id");
    const size_t n = (size_t)ctx->w * ctx->h;
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(ctx->hStageF, idepth, n * 4);
    memcpy(ctx->hStageF + n, idepthVar, n * 4);
    LSD_CHECK(ctx, cudaMemcpyAsync(s->idepth[0], ctx->hStageF, n * 4, cudaMemcpyHostToDevice, ctx->stream));
    LSD_CHECK(ctx, cudaMemcpyAsync(s->idepthVar[0], ctx->hStageF + n, n * 4, cudaMemcpyHostToDevice, ctx->stream));
    s->hasDepth = true; s->idepthPyrValid = false;
    return 0;
}

extern "C" int lsdgpu_frame_set_idepth_device(lsdgpu_ctx* ctx, int frame_id, const float* d_idepth, const float* d_idepthVar,
                                              size_t pitch, void* stream)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return failMissing(ctx, frame_id, "unknown frame id");
    int r = checkDevicePlaneF32(ctx, "frame_set_idepth_device", "the idepth", d_idepth, pitch);
    if (r || (r = checkDevicePlaneF32(ctx, "frame_set_idepth_device", "the idepthVar", d_idepthVar, pitch))) return r;
    const size_t row = (size_t)ctx->w * 4;
    LSD_CHECK(ctx, afterCallerStream(ctx, stream));
    LSD_CHECK(ctx, cudaMemcpy2DAsync(s->idepth[0], row, d_idepth, pitch, row, ctx->h, cudaMemcpyDefault, ctx->stream));
    LSD_CHECK(ctx, cudaMemcpy2DAsync(s->idepthVar[0], row, d_idepthVar, pitch, row, ctx->h, cudaMemcpyDefault, ctx->stream));
    LSD_CHECK(ctx, beforeCallerStream(ctx, stream));
    s->hasDepth = true; s->idepthPyrValid = false;
    return 0;
}

extern "C" int lsdgpu_frame_set_pose(lsdgpu_ctx* ctx, int frame_id, const double qts[8], int parent_id, float itr)
{ LSD_LOCK(ctx);
    FrameSlot* s = findFrame(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    memcpy(s->thisToParent, qts, sizeof(s->thisToParent));
    s->parentId = parent_id; s->initialTrackedResidual = itr;
    return 0;
}
extern "C" int lsdgpu_frame_get_pose(lsdgpu_ctx* ctx, int frame_id, double qts[8], int* parent_id, float* itr)
{ LSD_LOCK(ctx);
    FrameSlot* s = findFrame(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    if (qts) memcpy(qts, s->thisToParent, sizeof(s->thisToParent));
    if (parent_id) *parent_id = s->parentId;
    if (itr) *itr = s->initialTrackedResidual;
    return 0;
}
extern "C" int lsdgpu_frame_get_counters(lsdgpu_ctx* ctx, int frame_id, int* tracked, int* mapped)
{ LSD_LOCK(ctx);
    FrameSlot* s = findFrame(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    if (tracked) *tracked = s->numFramesTrackedOnThis;
    if (mapped) *mapped = s->numMappedOnThis;
    return 0;
}
extern "C" int lsdgpu_frame_set_counters(lsdgpu_ctx* ctx, int frame_id, int tracked, int mapped)
{ LSD_LOCK(ctx);
    FrameSlot* s = findFrame(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    s->numFramesTrackedOnThis = tracked; s->numMappedOnThis = mapped;
    return 0;
}
extern "C" int lsdgpu_frame_get_depth_stats(lsdgpu_ctx* ctx, int frame_id, float* meanIdepth, int* numPoints, int* flag)
{ LSD_LOCK(ctx);
    FrameSlot* s = findFrame(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    if ((meanIdepth || numPoints) && s->statsPending) {      // fetched lazily: keeps updateKeyframe free of host syncs
        LSD_CHECK(ctx, cudaSetDevice(ctx->device));
        LSD_CHECK(ctx, cudaMemcpyAsync(ctx->hScalars, s->dStats, 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
        s->numPoints = (int)ctx->hScalars[1];
        s->meanIdepth = (float)ctx->hScalars[0] / (float)s->numPoints;     // Frame.cpp:234
        s->statsPending = false;
    }
    if (meanIdepth) *meanIdepth = s->meanIdepth;
    if (numPoints) *numPoints = s->numPoints;
    if (flag) *flag = s->depthHasBeenUpdatedFlag ? 1 : 0;
    return 0;
}
extern "C" int lsdgpu_frame_clear_good_mask(lsdgpu_ctx* ctx, int frame_id)
{ LSD_LOCK(ctx);
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return failMissing(ctx, frame_id, "unknown frame id");
    s->hasGoodMask = false;
    return 0;
}

extern "C" int lsdgpu_ref_import(lsdgpu_ctx* ctx, int kf_id)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return failMissing(ctx, kf_id, "unknown keyframe id");
    int r = ensureIdepthPyramid(ctx, kf);
    if (r) return r;
    kf->depthHasBeenUpdatedFlag = false;       // SlamSystem.cpp:907-912
    return 0;
}

// ------------------------------------------------------------------------------------------------------
// input staging: UndistorterPTAM (SURVEY 8f row 3)
// ------------------------------------------------------------------------------------------------------
// Output camera of UndistorterPTAM for the "crop" / "full" / explicit modes and the remap tables (Undistorter.cpp:171-317).
// The expressions keep the reference's float / double mixing (int and 0.5 literals promote as written there); math calls on
// float arguments use the float overloads.
extern "C" int lsdgpu_undistorter_ptam_prepare(const float ic[5], int iw, int ih, const float ocIn[5], int ow, int oh,
                                               float* remapX, float* remapY, float K_out[9])
{
    if (!ic || !ocIn || iw <= 0 || ih <= 0 || ow <= 0 || oh <= 0) return -2;
    const float dist = ic[4];
    const float d2t = 2.0f * tanf(dist / 2.0f);
    float fx = ic[0] * iw, fy = ic[1] * ih;
    float cx = (float)((double)(ic[2] * iw) - 0.5), cy = (float)((double)(ic[3] * ih) - 0.5);
    // the reference rescales by in_width / in_width == 1.0 in double (:187-192): exact no-ops, including (c + 0.5) - 0.5
    auto undistRadius = [&](float r) { return tanf(r * dist) / d2t; };
    float ofx, ofy, ocx, ocy;
    if (ic[4] == 0) {
        ofx = ic[0] * ow; ofy = ic[1] * oh;
        ocx = (float)((double)(ic[2] * ow) - 0.5); ocy = (float)((double)(ic[3] * oh) - 0.5);
    } else if (ocIn[0] == -1 || ocIn[0] == -2) {
        const float rl = cx / fx, rr = (iw - 1 - cx) / fx, rt = cy / fy, rb = (ih - 1 - cy) / fy;
        const float sx = (float)ow / (float)iw, sy = (float)oh / (float)ih;
        if (ocIn[0] == -1) {            // "crop": the axis-aligned extremes
            const float tl = undistRadius(rl), tr = undistRadius(rr), tt = undistRadius(rt), tb = undistRadius(rb);
            ofy = fy * ((rt + rb) / (tt + tb)) * sy;
            ocy = (tt / rt) * ofy * cy / fy;
            ofx = fx * ((rl + rr) / (tl + tr)) * sx;
            ocx = (tl / rl) * ofx * cx / fx;
        } else {                        // "full": the four corners
            const float c_tl = sqrtf(rl * rl + rt * rt), c_tr = sqrtf(rr * rr + rt * rt);
            const float c_bl = sqrtf(rl * rl + rb * rb), c_br = sqrtf(rr * rr + rb * rb);
            const float u_tl = undistRadius(c_tl), u_tr = undistRadius(c_tr), u_bl = undistRadius(c_bl), u_br = undistRadius(c_br);
            // std::max(a, b) is `a < b ? b : a` (not fmaxf): a NaN first argument wins, a NaN second one loses.  With cx or
            // cy == 0 a corner radius is 0 and u / c is 0/0; the reference's ocy (or ocx) is then NaN and every entry -1.
            const auto stdMax = [](float a, float b) { return a < b ? b : a; };
            const float hor = stdMax(c_br, c_tr) + stdMax(c_bl, c_tl), vert = stdMax(c_tr, c_tl) + stdMax(c_bl, c_br);
            const float uhor = stdMax(u_br, u_tr) + stdMax(u_bl, u_tl), uvert = stdMax(u_tr, u_tl) + stdMax(u_bl, u_br);
            ofy = fy * ((vert) / (uvert)) * sy;
            ocy = stdMax(u_tl / c_tl, u_tr / c_tr) * ofy * cy / fy;
            ofx = fx * ((hor) / (uhor)) * sx;
            ocx = stdMax(u_bl / c_bl, u_tl / c_tl) * ofx * cx / fx;
        }
    } else {
        ofx = ocIn[0] * ow; ofy = ocIn[1] * oh;
        ocx = (float)((double)(ocIn[2] * ow) - 0.5); ocy = (float)((double)(ocIn[3] * oh) - 0.5);
    }
    // outputCalibration (:268-272) and K_ as main_on_images.cpp:164-167 reads it back
    const float oc0 = ofx / ow, oc1 = ofy / oh;
    const float oc2 = (float)(((double)ocx + 0.5) / ow), oc3 = (float)(((double)ocy + 0.5) / oh);
    if (K_out) {
        for (int i = 0; i < 9; i++) K_out[i] = 0.f;
        K_out[0] = oc0 * ow; K_out[4] = oc1 * oh;
        K_out[2] = (float)((double)(oc2 * ow) - 0.5); K_out[5] = (float)((double)(oc3 * oh) - 0.5);
        K_out[8] = 1.f;
    }
    if (remapX && remapY)
        for (int y = 0; y < oh; y++)
            for (int x = 0; x < ow; x++) {
                float ix = (x - ocx) / ofx, iy = (y - ocy) / ofy;
                const float r = sqrtf(ix * ix + iy * iy);
                const float fac = (r == 0 || dist == 0) ? 1 : atanf(r * d2t) / (dist * r);
                ix = fx * fac * ix + cx;
                iy = fy * fac * iy + cy;
                // "make rounding resistant" (:299-303; the last line assigns ix in the reference, kept)
                if (ix == 0) ix = (float)0.01;
                if (iy == 0) iy = (float)0.01;
                if (ix == iw - 1) ix = (float)(iw - 1.01);
                if (iy == ih - 1) ix = (float)(ih - 1.01);
                const bool inside = ix > 0 && iy > 0 && ix < iw - 1 && iy < ih - 1;
                remapX[x + y * ow] = inside ? ix : -1.f;
                remapY[x + y * ow] = inside ? iy : -1.f;
            }
    return (ih == oh && iw == ow && ic[4] == 0) ? 1 : 0;
}

extern "C" int lsdgpu_undistorter_validate_tables(int in_width, int in_height, int out_width, int out_height, const float* remapX, const float* remapY)
{
    if (!remapX || !remapY || in_width < 2 || in_height < 2 || out_width <= 0 || out_height <= 0) return -2;
    const long long n = (long long)out_width * out_height;
    for (long long i = 0; i < n; i++) {
        const float x = remapX[i], y = remapY[i];
        if (x < 0) continue;                                               // undistort() writes 0 (Undistorter.cpp:389-390)
        if (!(x >= 0 && y >= 0 && x < in_width - 1 && y < in_height - 1)) return (int)(1 + (i < 0x7ffffffeLL ? i : 0x7ffffffeLL));   // also NaN
    }
    return 0;
}

// frees the tables of whichever model is installed and the raw staging (the stream must be idle)
static void releaseUndistorter(lsdgpu_ctx* ctx)
{
    if (ctx->dRemapX) { cudaFree(ctx->dRemapX); ctx->dRemapX = nullptr; }
    if (ctx->dRemapY) { cudaFree(ctx->dRemapY); ctx->dRemapY = nullptr; }
    if (ctx->dCvMap1) { cudaFree(ctx->dCvMap1); ctx->dCvMap1 = nullptr; }
    if (ctx->dCvMap2) { cudaFree(ctx->dCvMap2); ctx->dCvMap2 = nullptr; }
    if (ctx->dRaw) { cudaFree(ctx->dRaw); ctx->dRaw = nullptr; }
    if (ctx->hRaw) { cudaFreeHost(ctx->hRaw); ctx->hRaw = nullptr; }
    ctx->undistorterSet = false;
}

extern "C" int lsdgpu_set_undistorter(lsdgpu_ctx* ctx, int in_width, int in_height, const float* remapX, const float* remapY)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (in_width <= 0 || in_height <= 0) return lsd_fail(ctx, "bad input size");
    const size_t n = (size_t)ctx->w * ctx->h, nr = (size_t)in_width * in_height;
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    releaseUndistorter(ctx);
    if (!remapX || !remapY) {
        if (in_width != ctx->w || in_height != ctx->h) return lsd_fail(ctx, "pass-through undistorter needs input size == context size");
    } else {
        if (lsdgpu_undistorter_validate_tables(in_width, in_height, ctx->w, ctx->h, remapX, remapY) != 0)
            return lsd_fail(ctx, "remap table entry outside the input image (lsdgpu_undistorter_validate_tables)");
        LSD_CHECK(ctx, cudaMalloc((void**)&ctx->dRemapX, n * 4));
        LSD_CHECK(ctx, cudaMalloc((void**)&ctx->dRemapY, n * 4));
        LSD_CHECK(ctx, cudaMemcpy(ctx->dRemapX, remapX, n * 4, cudaMemcpyHostToDevice));
        LSD_CHECK(ctx, cudaMemcpy(ctx->dRemapY, remapY, n * 4, cudaMemcpyHostToDevice));
    }
    LSD_CHECK(ctx, cudaMalloc((void**)&ctx->dRaw, nr));
    LSD_CHECK(ctx, cudaHostAlloc((void**)&ctx->hRaw, nr, cudaHostAllocDefault));
    ctx->rawW = in_width; ctx->rawH = in_height;
    ctx->undistorterSet = true;
    return 0;
}

static int uploadRaw(lsdgpu_ctx* ctx, const uint8_t* raw)
{
    if (!ctx->undistorterSet) return lsd_fail(ctx, "no undistorter installed (lsdgpu_set_undistorter)");
    const size_t nr = (size_t)ctx->rawW * ctx->rawH;
    cudaPointerAttributes pa;
    const bool pinned = cudaPointerGetAttributes(&pa, raw) == cudaSuccess && pa.type == cudaMemoryTypeHost;
    if (!pinned) {
        cudaGetLastError();
        LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));          // the previous raw image may still be in flight
        memcpy(ctx->hRaw, raw, nr);
    }
    LSD_CHECK(ctx, cudaMemcpyAsync(ctx->dRaw, pinned ? raw : ctx->hRaw, nr, cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

extern "C" int lsdgpu_undistort_u8(lsdgpu_ctx* ctx, const uint8_t* raw, uint8_t* out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    int r = uploadRaw(ctx, raw);
    if (r) return r;
    const int n = ctx->w * ctx->h;
    if (!ctx->dRemapX && !ctx->dCvMap1) {                             // result = image, Undistorter.cpp:370-375
        LSD_CHECK(ctx, cudaMemcpyAsync(out, ctx->dRaw, n, cudaMemcpyDeviceToHost, ctx->stream));
    } else {
        uint8_t* dOut = ctx->dStageU8[ctx->stageIdx];
        LSD_CHECK(ctx, cudaEventSynchronize(ctx->stageDone[ctx->stageIdx]));
        if (ctx->dCvMap1)
            k_undistort_opencv<<<divUp(n, 256), 256, 0, ctx->stream>>>(ctx->dRaw, ctx->rawW, ctx->rawH, ctx->dCvMap1, ctx->dCvMap2, n, dOut);
        else
            k_undistort<<<divUp(n, 256), 256, 0, ctx->stream>>>(ctx->dRaw, ctx->rawW, ctx->dRemapX, ctx->dRemapY, n, dOut);
        LAUNCH(ctx);
        LSD_CHECK(ctx, cudaGetLastError());
        LSD_CHECK(ctx, cudaMemcpyAsync(out, dOut, n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int lsdgpu_frame_upload_distorted_u8(lsdgpu_ctx* ctx, int frame_id, const uint8_t* raw)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s = acquireSlot(ctx, frame_id);
    if (!s) return failMissing(ctx, frame_id, "no free frame slot (release frames or raise max_frames)");
    int r = uploadRaw(ctx, raw);
    if (r) return r;
    return buildFrameFromDeviceU8(ctx, s, ctx->dRaw, ctx->rawW, ctx->dCvMap1 ? PYR_OPENCV : ctx->dRemapX ? PYR_PTAM : PYR_U8);
}

extern "C" int lsdgpu_frame_upload_distorted_device_u8(lsdgpu_ctx* ctx, int frame_id, const uint8_t* d_raw, size_t pitch, void* stream)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (!ctx->undistorterSet) return lsd_fail(ctx, "no undistorter installed (lsdgpu_set_undistorter)");
    int r = checkDeviceImage(ctx, "frame_upload_distorted_device_u8", d_raw, pitch, ctx->rawW, ctx->rawH);
    if (r) return r;
    FrameSlot* s = acquireSlot(ctx, frame_id);
    if (!s) return failMissing(ctx, frame_id, "no free frame slot (release frames or raise max_frames)");
    LSD_CHECK(ctx, afterCallerStream(ctx, stream));
    if ((r = buildFrameFromDeviceU8(ctx, s, d_raw, (int)pitch, ctx->dCvMap1 ? PYR_OPENCV : ctx->dRemapX ? PYR_PTAM : PYR_U8))) return r;
    LSD_CHECK(ctx, beforeCallerStream(ctx, stream));
    return 0;
}

// ------------------------------------------------------------------------------------------------------
// input staging: UndistorterOpenCV
// ------------------------------------------------------------------------------------------------------
// The constructor UndistorterOpenCV::UndistorterOpenCV (util/Undistorter.cpp:449-558) after parsing: cv::getOptimalNewCameraMatrix
// and cv::initUndistortRectifyMap(.., CV_16SC2) restated as OpenCV 4.13 computes them for the 4-coefficient model (no rotation,
// no tilt, no rational / thin-prism terms: the zero terms of OpenCV's general expressions are left out, which changes no bit
// of finite results).  All arithmetic is double, in OpenCV's order of operations.
namespace {
// cvRound / saturate_cast<int>(double): round half to even; out of range (and NaN) gives INT_MIN as cvtsd2si does
int cvRoundD(double v)
{
    return (v > -2147483648.5 && v < 2147483647.5) ? (int)std::nearbyint(v) : INT_MIN;
}
short saturateShort(int v) { return (short)(v < -32768 ? -32768 : v > 32767 ? 32767 : v); }
}

extern "C" int lsdgpu_undistorter_opencv_prepare(const float input_calibration[8], int iw, int ih, int output_mode, int ow, int oh,
                                                 int16_t* map1, uint16_t* map2, double K_new[9], float K_out[9])
{
    if (!input_calibration || iw <= 0 || ih <= 0 || ow <= 0 || oh <= 0) return -2;
    if (output_mode != -1 && output_mode != -2) return -2;         // "none" and explicit output parameters: valid = false (:493-502)
    float ic[8];
    for (int i = 0; i < 8; i++) ic[i] = input_calibration[i];
    if (ic[2] < 1.0f) {                                             // relative units (:519-534), in float as written
        ic[0] *= iw; ic[2] *= iw;
        ic[1] *= ih; ic[3] *= ih;
    }
    // originalK_ (CV_64F from the floats) and distCoeffs (CV_32F 4x1, converted to double by OpenCV)
    const double fx = ic[0], fy = ic[1], cx = ic[2], cy = ic[3];
    const double k1 = ic[4], k2 = ic[5], p1 = ic[6], p2 = ic[7];
    const double alpha = output_mode == -2 ? 1 : 0;

    // getOptimalNewCameraMatrix(K, D, in_size, alpha, out_size, nullptr, false): undistortPoints of a 9x9 grid over the input image
    // (fixed 5 iterations, with the icdist < 0 fallback of OpenCV 4.x), inscribed and circumscribed rectangles, alpha blend.  With
    // strong distortion the grid folds (interior points land outside the border); 4.13 then still frames the border.
    const int N = 9;
    const double ifx = 1. / fx, ify = 1. / fy;
    double iX0 = -FLT_MAX, iX1 = FLT_MAX, iY0 = -FLT_MAX, iY1 = FLT_MAX;
    double oX0 = FLT_MAX, oX1 = -FLT_MAX, oY0 = FLT_MAX, oY1 = -FLT_MAX;
    for (int gy = 0; gy < N; gy++)
        for (int gx = 0; gx < N; gx++) {
            const double u = (double)gx * (iw - 1) / (N - 1), v = (double)gy * (ih - 1) / (N - 1);
            double x = (u - cx) * ifx, y = (v - cy) * ify;
            const double x0 = x, y0 = y;
            for (int j = 0; j < 5; j++) {
                const double r2 = x * x + y * y;
                const double icdist = 1 / (1 + (k2 * r2 + k1) * r2);
                if (icdist < 0) {
                    x = (u - cx) * ifx;
                    y = (v - cy) * ify;
                    break;
                }
                const double deltaX = 2 * p1 * x * y + p2 * (r2 + 2 * x * x);
                const double deltaY = p1 * (r2 + 2 * y * y) + 2 * p2 * x * y;
                x = (x0 - deltaX) * icdist;
                y = (y0 - deltaY) * icdist;
            }
            if (gx == 0 || gx == N - 1 || gy == 0 || gy == N - 1) {   // 4.13: the circumscribed rectangle bounds the border points only
                oX0 = std::min(oX0, x); oX1 = std::max(oX1, x);
                oY0 = std::min(oY0, y); oY1 = std::max(oY1, y);
            }
            if (gx == 0) iX0 = std::max(iX0, x);
            if (gx == N - 1) iX1 = std::min(iX1, x);
            if (gy == 0) iY0 = std::max(iY0, y);
            if (gy == N - 1) iY1 = std::min(iY1, y);
        }
    const double fx0 = (ow - 1) / (iX1 - iX0), fy0 = (oh - 1) / (iY1 - iY0), cx0 = -fx0 * iX0, cy0 = -fy0 * iY0;
    const double fx1 = (ow - 1) / (oX1 - oX0), fy1 = (oh - 1) / (oY1 - oY0), cx1 = -fx1 * oX0, cy1 = -fy1 * oY0;
    double M[9] = { fx0 * (1 - alpha) + fx1 * alpha, 0, cx0 * (1 - alpha) + cx1 * alpha,
                    0, fy0 * (1 - alpha) + fy1 * alpha, cy0 * (1 - alpha) + cy1 * alpha,
                    0, 0, 1 };
    if (K_new) for (int i = 0; i < 9; i++) K_new[i] = M[i];
    if (K_out) {                                                    // K_ = K_new transposed (:557), read back by main_on_images.cpp:164-167
        for (int i = 0; i < 9; i++) K_out[i] = 0.f;
        K_out[0] = (float)M[0]; K_out[2] = (float)M[2];
        K_out[4] = (float)M[4]; K_out[5] = (float)M[5];
        K_out[8] = 1.f;
    }
    if (!map1 || !map2) return 0;

    // initUndistortRectifyMap(K, D, I, K_new, out_size, CV_16SC2): iR = K_new^-1 by cv::invert's 3x3 DECOMP_LU branch (cofactors
    // times 1 / det3), then per pixel the normalised ray, the distortion, the projection and 5-bit fixed point
    const double det = M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
    if (det == 0) return -2;
    const double d = 1. / det;
    const double ir[9] = { (M[4] * M[8] - M[5] * M[7]) * d, (M[2] * M[7] - M[1] * M[8]) * d, (M[1] * M[5] - M[2] * M[4]) * d,
                           (M[5] * M[6] - M[3] * M[8]) * d, (M[0] * M[8] - M[2] * M[6]) * d, (M[2] * M[3] - M[0] * M[5]) * d,
                           (M[3] * M[7] - M[4] * M[6]) * d, (M[1] * M[6] - M[0] * M[7]) * d, (M[0] * M[4] - M[1] * M[3]) * d };
    // The row walk is OpenCV's AVX2 one: the ray (X, Y, W) advances by 8 * ir[0..] per block of 8 pixels and is offset by k * ir[0..]
    // inside a block; a scalar tail (out_width % 8 pixels) advances pixel by pixel.  The walk only changes the last bits of the
    // ray, which reach the maps where a pixel projects ~1e7 px or more outside the image (a folded "full" view), never elsewhere.
    auto pixel = [&](int i, int j, double X, double Y, double W) {
        const double w = 1. / W, x = X * w, y = Y * w;
        const double x2 = x * x, y2 = y * y;
        const double r2 = x2 + y2, _2xy = 2 * x * y;
        const double kr = 1 + (k2 * r2 + k1) * r2;
        const double xd = x * kr + p1 * _2xy + p2 * (r2 + 2 * x2);
        const double yd = y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy;
        const double u = fx * xd + cx, v = fy * yd + cy;
        const int iu = cvRoundD(u * 32.0), iv = cvRoundD(v * 32.0);
        const size_t o = (size_t)i * ow + j;
        map1[2 * o] = saturateShort(iu >> 5);
        map1[2 * o + 1] = saturateShort(iv >> 5);
        map2[o] = (uint16_t)((iv & 31) * 32 + (iu & 31));
    };
    for (int i = 0; i < oh; i++) {
        double _x = i * ir[1] + ir[2], _y = i * ir[4] + ir[5], _w = i * ir[7] + ir[8];
        int j = 0;
        for (; j <= ow - 8; j += 8, _x += 8 * ir[0], _y += 8 * ir[3], _w += 8 * ir[6])
            for (int k = 0; k < 8; k++) pixel(i, j + k, _x + k * ir[0], _y + k * ir[3], _w + k * ir[6]);
        for (; j < ow; j++, _x += ir[0], _y += ir[3], _w += ir[6]) pixel(i, j, _x, _y, _w);
    }
    return 0;
}

extern "C" int lsdgpu_set_undistorter_opencv(lsdgpu_ctx* ctx, int in_width, int in_height, const int16_t* map1, const uint16_t* map2)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (in_width <= 0 || in_height <= 0) return lsd_fail(ctx, "bad input size");
    if (!map1 || !map2) return lsd_fail(ctx, "UndistorterOpenCV needs both maps");
    const size_t n = (size_t)ctx->w * ctx->h, nr = (size_t)in_width * in_height;
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    releaseUndistorter(ctx);
    LSD_CHECK(ctx, cudaMalloc((void**)&ctx->dCvMap1, n * sizeof(short2)));
    LSD_CHECK(ctx, cudaMalloc((void**)&ctx->dCvMap2, n * sizeof(uint16_t)));
    LSD_CHECK(ctx, cudaMemcpy(ctx->dCvMap1, map1, n * sizeof(short2), cudaMemcpyHostToDevice));
    LSD_CHECK(ctx, cudaMemcpy(ctx->dCvMap2, map2, n * sizeof(uint16_t), cudaMemcpyHostToDevice));
    LSD_CHECK(ctx, cudaMalloc((void**)&ctx->dRaw, nr));
    LSD_CHECK(ctx, cudaHostAlloc((void**)&ctx->hRaw, nr, cudaHostAllocDefault));
    ctx->rawW = in_width; ctx->rawH = in_height;
    ctx->undistorterSet = true;
    return 0;
}
