// records.cu -- frame memory of the C ABI (include/lsdgpu.h, DESIGN.md section 3): Frame::minimizeInMemory, FrameMemory::activateFrame
// + Frame::require, and the host records of minimized frames.  A minimized frame's record lives in the stream-ordered pools of two
// tiers, device and host memory; which frames move where is the caller's choice.
#include "internal.cuh"

// The buffers of a frame that a minimized record keeps, in record order: dStats, image / idepth / idepthVar of level 0, the
// reactivation data, the permaRef.  Buffers the frame does not have are null.  TIER_HOST: the part moves to the host body when the
// record is offloaded; the others (the device residue) are what the permaRef batches and the pending depth statistics read.
static int recordParts(const lsdgpu_ctx* ctx, FrameSlot& s, RecordPart* p)
{
    const size_t n0 = (size_t)ctx->w * ctx->h;
    int k = 0;
    p[k++] = { (char**)&s.dStats, 3 * sizeof(double), TIER_DEVICE };
    p[k++] = { (char**)&s.image[0], n0 * 4, TIER_HOST };
    p[k++] = { (char**)&s.idepth[0], s.hasDepth ? n0 * 4 : 0, TIER_HOST };
    p[k++] = { (char**)&s.idepthVar[0], s.hasDepth ? n0 * 4 : 0, TIER_HOST };
    p[k++] = { (char**)&s.reactIdepth, s.reactValid ? n0 * 4 : 0, TIER_HOST };
    p[k++] = { (char**)&s.reactVar, s.reactValid ? n0 * 4 : 0, TIER_HOST };
    p[k++] = { (char**)&s.reactValidity, s.reactValid ? n0 : 0, TIER_HOST };
    p[k++] = { (char**)&s.permaPC, (size_t)s.permaNumPts * 16, TIER_DEVICE };
    p[k++] = { (char**)&s.permaVar, (size_t)s.permaNumPts * 4, TIER_DEVICE };
    return k;
}

// Lays frame view `f`'s record out over blocks base[tier] (without `split`, the device block alone): each part in recordParts order
// at the next 256-byte boundary, absent parts null; bytes[t] = the size of block t.  base == nullptr only measures.
static void layoutRecord(const lsdgpu_ctx* ctx, FrameSlot& f, bool split, char* const* base, size_t bytes[TIERS])
{
    RecordPart p[REC_PARTS];
    const int np = recordParts(ctx, f, p);
    bytes[TIER_DEVICE] = bytes[TIER_HOST] = 0;
    for (int k = 0; k < np; k++) {
        const int b = split ? p[k].tier : TIER_DEVICE;
        if (base) *p[k].ptr = p[k].bytes ? base[b] + bytes[b] : nullptr;
        bytes[b] += alignUp(p[k].bytes, 256);
    }
    if (base)
        for (int t = 0; t < TIERS; t++) { f.record[t] = base[t]; f.recordBytes[t] = bytes[t]; }
}

// One k_record_copy from the parts of view `from` to those of view `to`; activation leaves out level 0 (k_image_pyramid reads it)
static int copyRecord(lsdgpu_ctx* ctx, FrameSlot& from, FrameSlot& to, bool withImage0 = true)
{
    RecordPart src[REC_PARTS], dst[REC_PARTS];
    const int np = recordParts(ctx, from, src);
    recordParts(ctx, to, dst);
    for (int k = 0; k < np; k++)
        if (!withImage0 && src[k].ptr == (char**)&from.image[0]) src[k].bytes = 0;
    return launchRecordCopy(ctx, src, dst, np);
}

cudaError_t freeRecord(lsdgpu_ctx* ctx, const FrameSlot& m)
{
    cudaError_t e = cudaSuccess;
    for (int t = 0; t < TIERS && e == cudaSuccess; t++)
        if (m.record[t]) e = cudaFreeAsync(m.record[t], ctx->stream);
    return e;
}

// A stream-ordered pool of pinned memory at `type` / `id`, read / write for device `access` if >= 0.  Freed blocks stay mapped for
// the next allocation instead of going back at each synchronisation (which made every allocation map fresh memory on the stream).
static cudaError_t createPool(cudaMemPool_t* out, cudaMemLocationType type, int id, int access)
{
    cudaMemPoolProps pp = {};
    pp.allocType = cudaMemAllocationTypePinned;
    pp.location.type = type; pp.location.id = id;
    cudaMemPool_t pool;
    cudaError_t e = cudaMemPoolCreate(&pool, &pp);
    if (e != cudaSuccess) return e;
    cudaMemAccessDesc ad = {};
    ad.location.type = cudaMemLocationTypeDevice; ad.location.id = access;
    ad.flags = cudaMemAccessFlagsProtReadWrite;
    uint64_t keep = UINT64_MAX;
    if ((access >= 0 && (e = cudaMemPoolSetAccess(pool, &ad, 1)) != cudaSuccess) ||
        (e = cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep)) != cudaSuccess) {
        cudaMemPoolDestroy(pool);
        return e;
    }
    *out = pool;
    return cudaSuccess;
}
cudaError_t ensureRecordPool(lsdgpu_ctx* ctx)
{
    return ctx->pool[TIER_DEVICE] ? cudaSuccess : createPool(&ctx->pool[TIER_DEVICE], cudaMemLocationTypeDevice, ctx->device, -1);
}
// The host tier: pinned memory on the device's host NUMA node, mapped for the device, so that the kernels that read a record
// (k_record_copy, k_image_pyramid, the cloud export) read a host body over the bus unchanged.  Created on the first offload.
static cudaError_t ensureHostPool(lsdgpu_ctx* ctx)
{
    if (ctx->pool[TIER_HOST]) return cudaSuccess;
    int supported = 0, numa = 0;
    cudaError_t e = cudaDeviceGetAttribute(&supported, cudaDevAttrHostNumaMemoryPoolsSupported, ctx->device);
    if (e == cudaSuccess && !supported) e = cudaErrorNotSupported;
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&numa, cudaDevAttrHostNumaId, ctx->device);
    if (e != cudaSuccess) return e;
    return createPool(&ctx->pool[TIER_HOST], cudaMemLocationTypeHostNuma, numa < 0 ? 0 : numa, ctx->device);   // -1: no NUMA nodes
}

extern "C" int lsdgpu_frame_release(lsdgpu_ctx* ctx, int frame_id)
{ LSD_LOCK(ctx);
    if (FrameSlot* s = findSlot(ctx, frame_id)) {
        if (ctx->activeKf == frame_id) return lsd_fail(ctx, "frame is the active keyframe of the depth map");
        s->used = false; s->id = -1;
        return 0;
    }
    FrameSlot* m = findMinimized(ctx, frame_id);
    if (!m) return lsd_fail(ctx, "unknown frame id");
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    LSD_CHECK(ctx, freeRecord(ctx, *m));
    ctx->minimized.erase(ctx->minimized.begin() + (m - ctx->minimized.data()));
    // the pools keep freed records for later minimizes and offloads (see createPool); a released frame's memory goes back to the
    // device and the host, down to what the records still alive need
    size_t live[TIERS];
    lsdgpu_frame_memory_usage(ctx, nullptr, &live[TIER_DEVICE], nullptr, &live[TIER_HOST]);
    for (int t = 0; t < TIERS; t++)
        if (ctx->pool[t]) LSD_CHECK(ctx, cudaMemPoolTrimTo(ctx->pool[t], live[t]));
    return 0;
}

extern "C" int lsdgpu_frame_minimize(lsdgpu_ctx* ctx, int frame_id)
{ LSD_LOCK(ctx);
    if (findMinimized(ctx, frame_id)) return 0;
    FrameSlot* s = findSlot(ctx, frame_id);
    if (!s) return lsd_fail(ctx, "unknown frame id");
    if (ctx->activeKf == frame_id) return lsd_fail(ctx, "frame is the active keyframe of the depth map");
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    LSD_CHECK(ctx, ensureRecordPool(ctx));
    FrameSlot m = *s;
    size_t bytes[TIERS];
    layoutRecord(ctx, m, false, nullptr, bytes);
    char* rec[TIERS] = { nullptr, nullptr };
    LSD_CHECK(ctx, cudaMallocFromPoolAsync((void**)&rec[TIER_DEVICE], bytes[TIER_DEVICE], ctx->pool[TIER_DEVICE], ctx->stream));
    layoutRecord(ctx, m, false, rec, bytes);
    const int r = copyRecord(ctx, *s, m);
    if (r) { freeRecord(ctx, m); return r; }
    for (int l = 0; l < LSD_LEVELS; l++) {
        m.grad[l] = nullptr;
        if (l) m.image[l] = m.idepth[l] = m.idepthVar[l] = nullptr;
    }
    m.maxgrad = nullptr; m.goodMask = nullptr;
    m.idepthPyrValid = false;
    m.hasGoodMask = false;                                          // clear_refPixelWasGood, Frame.cpp:388
    ctx->minimized.push_back(m);
    s->used = false; s->id = -1;
    return 0;
}

extern "C" int lsdgpu_frame_activate(lsdgpu_ctx* ctx, int frame_id)
{ LSD_LOCK(ctx);
    if (findSlot(ctx, frame_id)) return 0;
    FrameSlot* m = findMinimized(ctx, frame_id);
    if (!m) return lsd_fail(ctx, "unknown frame id");
    FrameSlot* c = nullptr;
    for (auto& f : ctx->slots)
        if (!f.used) { c = &f; break; }
    if (!c) {
        ctx->err = "no free frame slot to activate frame " + std::to_string(frame_id) + " (minimize or release frames, or raise max_frames); it stays minimized";
        return -2;
    }
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot a = *m;
    for (int l = 0; l < LSD_LEVELS; l++)                           // the slot's buffers
        a.image[l] = c->image[l], a.grad[l] = c->grad[l], a.idepth[l] = c->idepth[l], a.idepthVar[l] = c->idepthVar[l];
    a.maxgrad = c->maxgrad; a.goodMask = c->goodMask; a.dStats = c->dStats;
    a.permaPC = c->permaPC; a.permaVar = c->permaVar;
    a.reactIdepth = c->reactIdepth; a.reactVar = c->reactVar; a.reactValidity = c->reactValidity;
    int r = copyRecord(ctx, *m, a, false);
    if (r || (r = buildImagePyramidFromRecord(ctx, &a, m->image[0]))) return r;
    LSD_CHECK(ctx, freeRecord(ctx, *m));
    for (int t = 0; t < TIERS; t++) { a.record[t] = nullptr; a.recordBytes[t] = 0; }
    a.used = true;
    a.idepthPyrValid = false;                                       // ensureIdepthPyramid rebuilds levels 1..4 on first use
    a.reactAllocated = a.reactValid;
    *c = a;
    ctx->minimized.erase(ctx->minimized.begin() + (m - ctx->minimized.data()));
    return 0;
}

extern "C" int lsdgpu_frame_offload(lsdgpu_ctx* ctx, int frame_id)
{ LSD_LOCK(ctx);
    FrameSlot* m = findMinimized(ctx, frame_id);
    if (!m) {
        if (!findSlot(ctx, frame_id)) return lsd_fail(ctx, "unknown frame id");
        ctx->err = "frame " + std::to_string(frame_id) + " is active: only a minimized frame can be offloaded (lsdgpu_frame_minimize it first)";
        return -2;
    }
    if (m->record[TIER_HOST]) return 0;
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot o = *m;
    size_t bytes[TIERS];                                            // the device residue and the host body
    layoutRecord(ctx, o, true, nullptr, bytes);
    char* base[TIERS] = { nullptr, nullptr };
    cudaError_t e = ensureHostPool(ctx);
    if (e == cudaSuccess) e = cudaMallocFromPoolAsync((void**)&base[TIER_HOST], bytes[TIER_HOST], ctx->pool[TIER_HOST], ctx->stream);
    if (e != cudaSuccess) {
        cudaGetLastError();
        ctx->err = "frame_offload: no host memory for frame " + std::to_string(frame_id) + " (" + cudaGetErrorString(e) +
                   "); it stays minimized in device memory";
        return -1;
    }
    e = cudaMallocFromPoolAsync((void**)&base[TIER_DEVICE], bytes[TIER_DEVICE], ctx->pool[TIER_DEVICE], ctx->stream);
    if (e != cudaSuccess) { cudaFreeAsync(base[TIER_HOST], ctx->stream); LSD_CHECK(ctx, e); }
    layoutRecord(ctx, o, true, base, bytes);
    const int r = copyRecord(ctx, *m, o);
    if (r) { freeRecord(ctx, o); return r; }
    LSD_CHECK(ctx, freeRecord(ctx, *m));
    *m = o;
    return 0;
}

extern "C" int lsdgpu_frame_memory_usage(lsdgpu_ctx* ctx, int* n_device, size_t* device_bytes, int* n_host, size_t* host_bytes)
{ LSD_LOCK(ctx);
    int n[TIERS] = { 0, 0 };
    size_t b[TIERS] = { 0, 0 };
    for (const auto& m : ctx->minimized) {
        n[m.record[TIER_HOST] ? TIER_HOST : TIER_DEVICE]++;
        for (int t = 0; t < TIERS; t++) b[t] += m.recordBytes[t];
    }
    if (n_device) *n_device = n[TIER_DEVICE];
    if (device_bytes) *device_bytes = b[TIER_DEVICE];
    if (n_host) *n_host = n[TIER_HOST];
    if (host_bytes) *host_bytes = b[TIER_HOST];
    return 0;
}
