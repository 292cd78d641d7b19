// frames.cu -- frame slots of the C ABI (include/lsdgpu.h): upload, the device prefetch ring, release, download, pose / counter
// setters and getters, depth import, and the input undistorter (UndistorterPTAM) in front of the frame construction.
#include "internal.cuh"
#include "frame.cuh"

static FrameSlot* acquireSlot(lsdgpu_ctx* ctx, int id)
{
    FrameSlot* s = findSlot(ctx, id);
    if (s) return s;
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
            fresh.permaNumPts = 0;
            fresh.reactAllocated = false; fresh.reactValid = false;
            c = fresh;
            return &c;
        }
    return nullptr;
}

static int buildFrameFromDeviceU8(lsdgpu_ctx* ctx, FrameSlot* s, const uint8_t* dsrc, bool remap = false);

extern "C" int lsdgpu_frame_upload_u8(lsdgpu_ctx* ctx, int frame_id, const uint8_t* gray)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s = acquireSlot(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "no free frame slot (release frames or raise max_frames)");
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
    int r = buildFrameFromDeviceU8(ctx, s, ctx->dStageU8[b]);
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
    if (!s) return lsd_fail(ctx, "no free frame slot (release frames or raise max_frames)");
    return buildFrameFromDeviceU8(ctx, s, ctx->stageRing + (size_t)index * ctx->w * ctx->h);
}

static int buildFrameFromDeviceU8(lsdgpu_ctx* ctx, FrameSlot* s, const uint8_t* dsrc, bool remap)
{
    const int w = ctx->w, h = ctx->h;
    PyrPtrs pp;
    for (int l = 0; l < LSD_LEVELS; l++) pp.l[l] = s->image[l];
    if (remap) k_image_pyramid<true><<<dim3(w / 16, h / 16), 256, 0, ctx->stream>>>(dsrc, pp, w, h, ctx->dRemapX, ctx->dRemapY, ctx->rawW, nullptr);
    else k_image_pyramid<false><<<dim3(w / 16, h / 16), 256, 0, ctx->stream>>>(dsrc, pp, w, h);
    LAUNCH(ctx);
    GradPtrs gp;
    for (int l = 0; l < LSD_LEVELS; l++) { gp.img[l] = s->image[l]; gp.grad[l] = s->grad[l]; gp.w[l] = w >> l; gp.h[l] = h >> l; }
    gp.maxgrad0 = s->maxgrad;
    // blockIdx.y = level; level 0 runs as 32x8 tiles, levels 1..4 linearly (their block counts are smaller than the tile count)
    LSD_CHECK(ctx, launchPDL(k_gradients, dim3(divUp(w, GR_TW) * divUp(h, GR_TH), LSD_LEVELS), dim3(256), 0, ctx->stream, gp));      // + maxGradients of level 0
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    s->hasDepth = false; s->idepthPyrValid = false; s->hasGoodMask = false;
    return 0;
}

extern "C" int lsdgpu_frame_release(lsdgpu_ctx* ctx, int frame_id)
{ LSD_LOCK(ctx);
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    if (ctx->activeKf == frame_id) return lsd_fail(ctx, "frame is the active keyframe of the depth map");
    s->used = false; s->id = -1;
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

extern "C" int lsdgpu_frame_download(lsdgpu_ctx* ctx, int frame_id, int what, int level, void* out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    if (level < 0 || level >= LSD_LEVELS) return lsd_fail(ctx, "bad level");
    const size_t n = ((size_t)ctx->w * ctx->h) >> (2 * level);
    const void* src = nullptr;
    size_t bytes = 0;
    switch (what) {
    case LSDGPU_BUF_IMAGE: src = s->image[level]; bytes = n * 4; break;
    case LSDGPU_BUF_GRADIENTS: src = s->grad[level]; bytes = n * 16; break;
    case LSDGPU_BUF_MAXGRAD: if (level != 0) return lsd_fail(ctx, "maxGradients exists at level 0 only"); src = s->maxgrad; bytes = n * 4; break;
    case LSDGPU_BUF_IDEPTH:
    case LSDGPU_BUF_IDEPTH_VAR:
        if (!s->hasDepth) return lsd_fail(ctx, "frame has no depth");
        if (level > 0) { int r = ensureIdepthPyramid(ctx, s); if (r) return r; }
        src = (what == LSDGPU_BUF_IDEPTH) ? s->idepth[level] : s->idepthVar[level]; bytes = n * 4; break;
    case LSDGPU_BUF_GOODMASK:
        if (!s->hasGoodMask) { memset(out, 1, ((size_t)ctx->w * ctx->h) / 4); return 0; }   // Frame.h:433: initialised to true
        src = s->goodMask; bytes = ((size_t)ctx->w * ctx->h) / 4; break;
    default: return lsd_fail(ctx, "bad buffer selector");
    }
    LSD_CHECK(ctx, cudaMemcpyAsync(out, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int lsdgpu_frame_set_depth_gt(lsdgpu_ctx* ctx, int frame_id, const float* depth, float cov_scale)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    const int n = ctx->w * ctx->h;
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(ctx->hStageF, depth, (size_t)n * 4);
    LSD_CHECK(ctx, cudaMemcpyAsync(ctx->dStageF, ctx->hStageF, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    k_set_depth_gt<<<divUp(n, 256), 256, 0, ctx->stream>>>(ctx->dStageF, s->maxgrad, s->idepth[0], s->idepthVar[0], ctx->w, ctx->h,
                                                           ctx->g.minUseGrad, cov_scale);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    s->hasDepth = true; s->idepthPyrValid = false;
    return 0;
}

extern "C" int lsdgpu_frame_set_idepth(lsdgpu_ctx* ctx, int frame_id, const float* idepth, const float* idepthVar)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    const size_t n = (size_t)ctx->w * ctx->h;
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(ctx->hStageF, idepth, n * 4);
    memcpy(ctx->hStageF + n, idepthVar, n * 4);
    LSD_CHECK(ctx, cudaMemcpyAsync(s->idepth[0], ctx->hStageF, n * 4, cudaMemcpyHostToDevice, ctx->stream));
    LSD_CHECK(ctx, cudaMemcpyAsync(s->idepthVar[0], ctx->hStageF + n, n * 4, cudaMemcpyHostToDevice, ctx->stream));
    s->hasDepth = true; s->idepthPyrValid = false;
    return 0;
}

extern "C" int lsdgpu_frame_set_pose(lsdgpu_ctx* ctx, int frame_id, const double qts[8], int parent_id, float itr)
{ LSD_LOCK(ctx);
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    memcpy(s->thisToParent, qts, sizeof(s->thisToParent));
    s->parentId = parent_id; s->initialTrackedResidual = itr;
    return 0;
}
extern "C" int lsdgpu_frame_get_pose(lsdgpu_ctx* ctx, int frame_id, double qts[8], int* parent_id, float* itr)
{ LSD_LOCK(ctx);
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    if (qts) memcpy(qts, s->thisToParent, sizeof(s->thisToParent));
    if (parent_id) *parent_id = s->parentId;
    if (itr) *itr = s->initialTrackedResidual;
    return 0;
}
extern "C" int lsdgpu_frame_get_counters(lsdgpu_ctx* ctx, int frame_id, int* tracked, int* mapped)
{ LSD_LOCK(ctx);
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    if (tracked) *tracked = s->numFramesTrackedOnThis;
    if (mapped) *mapped = s->numMappedOnThis;
    return 0;
}
extern "C" int lsdgpu_frame_set_counters(lsdgpu_ctx* ctx, int frame_id, int tracked, int mapped)
{ LSD_LOCK(ctx);
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    s->numFramesTrackedOnThis = tracked; s->numMappedOnThis = mapped;
    return 0;
}
extern "C" int lsdgpu_frame_get_depth_stats(lsdgpu_ctx* ctx, int frame_id, float* meanIdepth, int* numPoints, int* flag)
{ LSD_LOCK(ctx);
    FrameSlot* s = findSlot(ctx, frame_id);
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
    if (!s) return lsd_fail(ctx, "unknown frame id");
    s->hasGoodMask = false;
    return 0;
}

extern "C" int lsdgpu_ref_import(lsdgpu_ctx* ctx, int kf_id)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return lsd_fail(ctx, "unknown keyframe id");
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
            const float hor = fmaxf(c_br, c_tr) + fmaxf(c_bl, c_tl), vert = fmaxf(c_tr, c_tl) + fmaxf(c_bl, c_br);
            const float uhor = fmaxf(u_br, u_tr) + fmaxf(u_bl, u_tl), uvert = fmaxf(u_tr, u_tl) + fmaxf(u_bl, u_br);
            ofy = fy * ((vert) / (uvert)) * sy;
            ocy = fmaxf(u_tl / c_tl, u_tr / c_tr) * ofy * cy / fy;
            ofx = fx * ((hor) / (uhor)) * sx;
            ocx = fmaxf(u_bl / c_bl, u_tl / c_tl) * ofx * cx / fx;
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

extern "C" int lsdgpu_set_undistorter(lsdgpu_ctx* ctx, int in_width, int in_height, const float* remapX, const float* remapY)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (in_width <= 0 || in_height <= 0) return lsd_fail(ctx, "bad input size");
    const size_t n = (size_t)ctx->w * ctx->h, nr = (size_t)in_width * in_height;
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    if (ctx->dRemapX) { cudaFree(ctx->dRemapX); ctx->dRemapX = nullptr; }
    if (ctx->dRemapY) { cudaFree(ctx->dRemapY); ctx->dRemapY = nullptr; }
    if (ctx->dRaw) { cudaFree(ctx->dRaw); ctx->dRaw = nullptr; }
    if (ctx->hRaw) { cudaFreeHost(ctx->hRaw); ctx->hRaw = nullptr; }
    ctx->undistorterSet = false;
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
    if (!ctx->dRemapX) {                                              // result = image, Undistorter.cpp:370-375
        LSD_CHECK(ctx, cudaMemcpyAsync(out, ctx->dRaw, n, cudaMemcpyDeviceToHost, ctx->stream));
    } else {
        uint8_t* dOut = ctx->dStageU8[ctx->stageIdx];
        LSD_CHECK(ctx, cudaEventSynchronize(ctx->stageDone[ctx->stageIdx]));
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
    if (!s) return lsd_fail(ctx, "no free frame slot (release frames or raise max_frames)");
    int r = uploadRaw(ctx, raw);
    if (r) return r;
    return buildFrameFromDeviceU8(ctx, s, ctx->dRaw, ctx->dRemapX != nullptr);
}
