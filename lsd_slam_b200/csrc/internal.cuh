// internal.cuh -- context, device layouts and launch helpers of liblsdgpu (not part of the ABI).
//
// Data layout in HBM (DESIGN.md section 3):
//   * one arena per context, carved into `max_frames` frame slots + one depth map + tracker scratch;
//   * frame slot: image pyramid f32 planar L0..L4, gradient pyramid float4 (dx,dy,I,0) L0..L4,
//     maxGradients L0 f32, idepth / idepthVar pyramids f32 L0..L4, refPixelWasGood u8 at L1;
//   * depth map: two ping-pong copies (current / other) of the hypothesis field, each as two 16-byte planes
//       hf = float4(idepth, idepth_var, idepth_smoothed, idepth_var_smoothed)
//       hi = int4  (isValid, blacklisted, validity_counter, bits(nextStereoFrameMinID))
//     (the reference's 32-byte AoS record split in halves, so that every access is one 128-bit transaction),
//     plus the int32 validity integral image.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/lsdgpu.h"
#include "hostmath.h"

#define LSD_LEVELS LSDGPU_LEVELS
#define SE3TRACKING_MIN_LEVEL 1
#define SE3TRACKING_MAX_LEVEL 5

struct LevelCam {
    int w, h;
    float fx, fy, cx, cy;
    float fxi, fyi, cxi, cyi;
    float K[9], KInv[9];
};

enum { TIER_DEVICE = 0, TIER_HOST = 1, TIERS = 2 };     // the memory of a minimized frame's record: device, or host (records.cu)

struct FrameSlot {
    int id = -1;
    bool used = false;
    float* image[LSD_LEVELS];
    float4* grad[LSD_LEVELS];
    float* maxgrad;
    float* idepth[LSD_LEVELS];
    float* idepthVar[LSD_LEVELS];
    uint8_t* goodMask;
    float4* permaPC = nullptr;           // permaRef: (x, y, z, colour) per level-4 point (Frame::setPermaRef)
    float* permaVar = nullptr;
    int permaNumPts = 0;
    bool permaSet = false;               // setPermaRef ran (a keyframe without points has a permaRef of 0 points)
    float* reactIdepth = nullptr;        // Frame::idepth_reAct / idepthVar_reAct / validity_reAct (Frame.cpp:107-145), device-resident
    float* reactVar = nullptr;
    uint8_t* reactValidity = nullptr;
    bool reactAllocated = false, reactValid = false;
    bool hasDepth = false, idepthPyrValid = false, hasGoodMask = false;
    bool depthHasBeenUpdatedFlag = false;
    float meanIdepth = 1.f;
    int numPoints = 0;
    double* dStats = nullptr;            // device: sum(idepth_smoothed), count, rescale (written by setDepth kernels)
    bool statsPending = false;           // meanIdepth / numPoints still have to be fetched from dStats
    double thisToParent[8];
    int parentId = -1;
    float initialTrackedResidual = 0.f;
    int numFramesTrackedOnThis = 0, numMappedOnThis = 0;
    // minimized frame: its record's block per tier, which the pointers above point into.  An offloaded record (lsdgpu_frame_offload)
    // keeps the residue (dStats, the permaRef) in the device block and the body (level 0, the reactivation data) in the host block.
    char* record[TIERS] = { nullptr, nullptr };
    size_t recordBytes[TIERS] = { 0, 0 };
};
// a buffer of a frame that its minimized record keeps (recordParts, records.cu): the frame's pointer to it, its size, its tier
struct RecordPart { char** ptr; size_t bytes; int tier; };
#define REC_PARTS 9

struct PyrPtrs {
    float* l[LSD_LEVELS];
};

struct HypField {
    float4* hf;
    int4* hi;
};

// per reference-frame constants of Frame::prepareForStereoWith (Frame.cpp:295-317) + what observeDepth reads
struct RefConst {
    float K_otherToThis_R[9];
    float K_otherToThis_t[3];
    float otherToThis_t[3];
    float thisToOther_t[3];
    float row0[3], row1[3], row2[3];
    float initialTrackedResidual;
    int id;
    int trackedOnActive;          // refFrame->getTrackingParent() == activeKeyFrame
    const float* image;           // level 0
    const uint8_t* goodMask;      // refPixelWasGoodNoCreate() or nullptr
};
#define LSD_MAX_PERMA_BATCH 4096
#define LSD_MAX_REFS 16
#define LSD_MAX_ID_SPAN 64
#define SEQ_NBIN 24          // sequential fp32 sum (seqsum.cuh): binades 2^0 .. 2^23 are tabulated
#define SEQ_RUN 256          // pixels per tabulated run (one warp, 8 per lane)
struct ObserveParams {
    RefConst refs[LSD_MAX_REFS];
    int nRefs;
    int byIdOffset, byIdSize;     // referenceFrameByID_offset / size
    int byId[LSD_MAX_ID_SPAN];    // id - offset -> index into refs
    int oldestIdx, newestIdx;
    int reactivated;
    int kfNumTracked, kfNumMapped;
};

// number of reduction channels of one tracker evaluation (see track.cuh)
#define EV_NCH 40

// sizes of the random start's buffers (the generator itself is rand.cuh): glibc's 5 state types, polynomials / windows of up to
// 63 words padded to 64, per type 63 jump rows + 64 draw rows; the depth map is split into tiles of RND_TILE pixels
#define RND_TYPES 5
#define RND_ROW 64
#define RND_POW_ROWS 63
#define RND_GEN_ROWS 64
#define RND_TYPE_WORDS ((RND_POW_ROWS + RND_GEN_ROWS) * RND_ROW)
#define RND_TILE 1024

struct lsdgpu_ctx {
    // Every entry point of the C ABI holds this for its whole duration (LSD_LOCK): one context may be shared by SlamSystem's
    // tracking and mapping threads (SlamSystem.cpp:111, :206) -- their calls serialise here, as they do on the frame / keyframe
    // locks of the reference (Frame::getActiveLock, SE3Tracker.cpp:286, DepthMap.cpp:1104).  Recursive: the fused entry points
    // (lsdgpu_track_and_map, lsdgpu_sim3_track) call other entry points.
    mutable std::recursive_mutex mu;
    int device = 0;
    int w = 0, h = 0;
    LevelCam cam[LSD_LEVELS];
    lsdgpu_globals g;
    cudaStream_t stream = nullptr;
    std::string err;
    long long launches = 0;
    int smCount = 132;                   // H100 SXM; set from the device at context creation

    char* arena = nullptr;
    size_t arenaBytes = 0;
    std::vector<FrameSlot> slots;
    // minimized frames (Frame::minimizeInMemory): the frame's metadata, with image / idepth / idepthVar of level 0, the
    // reactivation data, the permaRef and dStats pointing into its record and every other device pointer null.  Records come in
    // stream order from the pool of their tier; the host tier is pinned memory on the device's host NUMA node (DESIGN.md section 3).
    std::vector<FrameSlot> minimized;
    cudaMemPool_t pool[TIERS] = { nullptr, nullptr };

    // depth map
    HypField cur, oth;
    int* integral = nullptr;
    int activeKf = -1;
    bool activeKfReactivated = false;
    ObserveParams hObs;                  // passed to k_observe by value (__grid_constant__)
    int* propHead = nullptr;             // per-target list heads (propagateDepth)
    int* propNext = nullptr;
    float4* propVal = nullptr;           // per-source (new_idepth, new_var, validity, -)
    double* dScalars = nullptr;          // small device scratch for reductions (sum, count)
    double* hScalars = nullptr;          // pinned mirror
    // DepthMap::initializeRandomly (lsdgpu_depth_init_random, rand.cuh): the generator's tables of all types (copied on first use),
    // per-tile draw counts then offsets, and the result (number of draws, then the window after the last draw)
    uint32_t* rndTab = nullptr;
    bool rndTabReady = false;
    int* rndTiles = nullptr;
    uint32_t* rndOut = nullptr;

    // tracker scratch
    float* evPartials = nullptr;         // [maxBlocks][EV_NCH]
    unsigned int* evCounter = nullptr;
    float* dEvOut = nullptr;             // EV_NCH floats (device)
    float* hEvOut = nullptr;             // pinned host mirror
    void* hTrackState = nullptr;         // mapped pinned result block of the persistent tracker (host view)
    void* dTrackStateMapped = nullptr;   // device view of the same block
    void* dPermaItems = nullptr;         // batched permaRef tracking: candidate descriptors / results (device)
    void* dPermaResults = nullptr;
    void* dSim3Items = nullptr;          // batched Sim3 tracking: problem descriptors / results (device)
    void* dSim3Outs = nullptr;
    float* dRemapX = nullptr;            // UndistorterPTAM remap tables (separate allocation), raw-image staging
    float* dRemapY = nullptr;
    short2* dCvMap1 = nullptr;           // UndistorterOpenCV remap maps (CV_16SC2 integer part, CV_16UC1 fractions), separate allocations
    uint16_t* dCvMap2 = nullptr;
    uint8_t* dRaw = nullptr;
    uint8_t* hRaw = nullptr;
    int rawW = 0, rawH = 0;
    bool undistorterSet = false;
    int inputFormat = LSDGPU_PIX_MONO8;  // pixel format of the raw images (lsdgpu_set_input_format); kept across undistorter installs
    uint32_t* dPacked = nullptr;         // keyframeMsg.pointcloud staging: w*h InputPointDense records (device)
    int trackGrid = 132;                 // launch shape of the persistent tracker (set by trackPersistentSetup): one CTA per SM
    unsigned int* trkSync = nullptr;     // barrier counters + cross-GPU exchange slots of the persistent tracker (TP_SYNC_WORDS)
    unsigned int trkBase = 0;            // arrivals already counted on the grid barrier's counter (never reset)
    // one stream sharded over several GPUs (lsdgpu_peer_attach): every rank's arena mapped into this process
    int nRanks = 1, rank = 0;
    char* peerBase[8] = { nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr };
    unsigned int trkTailBase = 0;
    // several contexts tracked in one launch (lsdgpu_track_and_map_group)
    uint8_t* dLastMask = nullptr;        // level-1 flags of the last candidate of a pass (w*h/4 bytes)
    void* dGroupSegs = nullptr;          // TP_MAX_GROUP segment descriptors of a group launched on this context's stream (device)
    void* hGroupSegs = nullptr;          // their pinned staging
    cudaEvent_t groupEvent = nullptr;    // orders the group launch after the other streams' work and their later work after it
    bool optTrackDebug = false;          // LSDGPU_TRACK_DEBUG, read once at lsdgpu_create
    int2* seqTable = nullptr;            // seqsum.cuh: per-run maps of the sequential fp32 sum, [SEQ_NBIN][runs]
    unsigned char* seqFlags = nullptr;
    int* seqCounts = nullptr;
    unsigned int trackSeq = 0;           // sequence number of the last tracking launch (TrackState::doneSeq)
    uint8_t* stageRing = nullptr;        // device prefetch ring of raw u8 frames (separate allocation)
    int stageEntries = 0;
    uint8_t* hStage[2] = { nullptr, nullptr };   // double-buffered pinned staging for the u8 frame upload
    uint8_t* dStageU8[2] = { nullptr, nullptr };
    cudaEvent_t stageDone[2];
    int stageIdx = 0;
    float* hStageF = nullptr;            // pinned float staging (depth / idepth uploads)
    float* dStageF = nullptr;
    // lsdgpu_map_export_pointcloud (cloud.cuh): separate allocations made by lsdgpu_cloud_reserve, two of each (batch b uses set b & 1)
    int cloudMaxKf = 0;
    char* cloudMem = nullptr;            // device: descriptors, tile states + ticket + counts, output points, intensity table
    char* hCloudMem = nullptr;           // pinned: descriptors and counts of both sets
    void* dCloudKfs[2] = { nullptr, nullptr };
    void* hCloudKfs[2] = { nullptr, nullptr };
    unsigned long long* dCloudState[2] = { nullptr, nullptr };   // tile states, then the ticket, then 2 counts per keyframe
    size_t cloudStateBytes = 0;
    int* hCloudCounts[2] = { nullptr, nullptr };
    float4* dCloudOut[2] = { nullptr, nullptr };
    float* dCloudIntensity = nullptr;
    cudaStream_t cloudCopyStream = nullptr;
    cudaEvent_t cloudKernDone[2], cloudCopyDone[2];
    cudaEvent_t cloudT0 = nullptr, cloudT1 = nullptr;
    bool cloudTimed = false;
    // the *_device entry points: callerIn orders the context's stream after the caller's stream, callerOut the caller's after it
    cudaEvent_t callerIn = nullptr, callerOut = nullptr;

    // timers
    cudaEvent_t tBegin[8], tEnd[8];
    cudaEvent_t kBegin, kEnd;
    double trackKernelMs = 0;
    long long trackKernelLaunches = 0;
    double trackKernelBytes = 0;
    bool profileTrackKernel = false;
    bool trackProfilePending = false;
};

struct CtxLock {
    std::recursive_mutex* m;
    explicit CtxLock(const lsdgpu_ctx* c) : m(c ? &c->mu : nullptr) { if (m) m->lock(); }
    ~CtxLock() { if (m) m->unlock(); }
    CtxLock(const CtxLock&) = delete;
};
#define LSD_LOCK(ctx) CtxLock lsd_lock_(ctx)

#define LAUNCH(ctx) ((ctx)->launches++)

#define LSD_CHECK(ctx, expr)                                                                              \
    do {                                                                                                  \
        cudaError_t _e = (expr);                                                                          \
        if (_e != cudaSuccess) {                                                                          \
            char _b[512];                                                                                 \
            snprintf(_b, sizeof(_b), "%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            (ctx)->err = _b;                                                                              \
            return -1;                                                                                    \
        }                                                                                                 \
    } while (0)

// Programmatic dependent launch (sm_90+): a kernel launched with LSD_PDL_LAUNCH may be scheduled while its predecessor in the stream
// is still running; it must not touch the predecessor's output before pdlWait() returns (griddepcontrol.wait: all memory operations
// of the predecessor grid are complete and visible).  With the wait as the kernel's first statement the stream semantics are
// unchanged; what is saved is the launch latency between dependent kernels of a step.
__device__ __forceinline__ void pdlWait()
{
    asm volatile("griddepcontrol.wait;" ::: "memory");
}
template <typename... KArgs, typename... Args>
static inline cudaError_t launchPDL(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

static inline int lsd_fail(lsdgpu_ctx* ctx, const char* msg)
{
    ctx->err = msg;
    return -2;
}

static inline FrameSlot* findSlot(lsdgpu_ctx* ctx, int id)
{
    for (auto& s : ctx->slots)
        if (s.used && s.id == id) return &s;
    return nullptr;
}

static inline FrameSlot* findMinimized(lsdgpu_ctx* ctx, int id)
{
    for (auto& s : ctx->minimized)
        if (s.id == id) return &s;
    return nullptr;
}
// a frame in a slot or minimized: the entry points that read a minimized frame's record in place
static inline FrameSlot* findFrame(lsdgpu_ctx* ctx, int id)
{
    FrameSlot* s = findSlot(ctx, id);
    return s ? s : findMinimized(ctx, id);
}
// the error of an entry point that needs frame `id` in a slot: `msg` when the id is unknown, or that the frame is minimized
static inline int failMissing(lsdgpu_ctx* ctx, int id, const char* msg)
{
    if (!findMinimized(ctx, id)) return lsd_fail(ctx, msg);
    ctx->err = "frame " + std::to_string(id) + " is minimized (lsdgpu_frame_activate it first)";
    return -2;
}

// ---- the *_device entry points (include/lsdgpu.h): the caller's stream and the caller's device pointers ------------------------
// NULL is the legacy default stream (the library's own default stream need not be the legacy one)
static inline cudaStream_t callerStream(void* stream) { return stream ? (cudaStream_t)stream : cudaStreamLegacy; }
// the context's next work starts after everything enqueued on the caller's stream so far
static inline cudaError_t afterCallerStream(lsdgpu_ctx* ctx, void* stream)
{
    cudaError_t e = cudaEventRecord(ctx->callerIn, callerStream(stream));
    return e != cudaSuccess ? e : cudaStreamWaitEvent(ctx->stream, ctx->callerIn, 0);
}
// the caller's later work on its stream starts after everything enqueued on the context's stream so far
static inline cudaError_t beforeCallerStream(lsdgpu_ctx* ctx, void* stream)
{
    cudaError_t e = cudaEventRecord(ctx->callerOut, ctx->stream);
    return e != cudaSuccess ? e : cudaStreamWaitEvent(callerStream(stream), ctx->callerOut, 0);
}
// 0 if p is device or managed memory of the context's device, aligned to `align` bytes; otherwise an error naming `what`
static inline int checkDevicePtr(lsdgpu_ctx* ctx, const char* fn, const char* what, const void* p, size_t align)
{
    char msg[256];
    cudaPointerAttributes pa;
    const cudaError_t e = p ? cudaPointerGetAttributes(&pa, p) : cudaErrorInvalidValue;
    if (e != cudaSuccess) cudaGetLastError();
    if (!p || e != cudaSuccess || (pa.type != cudaMemoryTypeDevice && pa.type != cudaMemoryTypeManaged)) {
        snprintf(msg, sizeof(msg), "%s: %s is not device memory", fn, what);
        return lsd_fail(ctx, msg);
    }
    if (pa.device != ctx->device) {
        snprintf(msg, sizeof(msg), "%s: %s is memory of device %d, the context's device is %d", fn, what, pa.device, ctx->device);
        return lsd_fail(ctx, msg);
    }
    if ((uintptr_t)p % align) {
        snprintf(msg, sizeof(msg), "%s: %s is not %zu-byte aligned", fn, what, align);
        return lsd_fail(ctx, msg);
    }
    return 0;
}
// a caller's device image of width x height bytes with row pitch `pitch` (the kernels index it with int arithmetic)
static inline int checkDeviceImage(lsdgpu_ctx* ctx, const char* fn, const uint8_t* p, size_t pitch, int width, int height)
{
    char msg[256];
    if (pitch < (size_t)width || pitch > (size_t)INT32_MAX / (size_t)height) {
        snprintf(msg, sizeof(msg), "%s: row pitch %zu bytes for an image %d bytes wide (%d rows)", fn, pitch, width, height);
        return lsd_fail(ctx, msg);
    }
    return checkDevicePtr(ctx, fn, "the image", p, 1);
}
// a caller's device plane of the context's w x h floats with row pitch `pitch` bytes: whole floats, at least w of them (the kernels
// index it in floats with int arithmetic)
static inline int checkDevicePlaneF32(lsdgpu_ctx* ctx, const char* fn, const char* what, const float* p, size_t pitch)
{
    char msg[256];
    if (pitch % 4 || pitch < (size_t)ctx->w * 4 || pitch / 4 > (size_t)INT32_MAX / (size_t)ctx->h) {
        snprintf(msg, sizeof(msg), "%s: row pitch %zu bytes for %s of %d floats per row (%d rows): needs a multiple of 4 >= %d",
                 fn, pitch, what, ctx->w, ctx->h, ctx->w * 4);
        return lsd_fail(ctx, msg);
    }
    return checkDevicePtr(ctx, fn, what, p, 4);
}
// 0 if a caller's output of `capacity` bytes holds the `need` bytes of `what`
static inline int checkCapacity(lsdgpu_ctx* ctx, const char* fn, const char* what, size_t need, size_t capacity)
{
    if (capacity >= need) return 0;
    char msg[192];
    snprintf(msg, sizeof(msg), "%s: %s has %zu bytes, the output holds %zu", fn, what, need, capacity);
    return lsd_fail(ctx, msg);
}

static inline int divUp(int a, int b) { return (a + b - 1) / b; }
static inline size_t alignUp(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---- host helpers shared by the units of the library (each defined once, in the unit named) ---------------------------
int ensureIdepthPyramid(lsdgpu_ctx* ctx, FrameSlot* s);     // frames.cu: levels 1..4 of a keyframe's idepth / idepthVar
// frames.cu, which compiles frame.cuh's kernels, launches them for records.cu: one k_record_copy of the parts from[k] -> to[k]
// that have bytes, and Frame::require's image pyramid and gradients of slot `s` from the fp32 level 0 of a record
int launchRecordCopy(lsdgpu_ctx* ctx, const RecordPart* from, const RecordPart* to, int n);
int buildImagePyramidFromRecord(lsdgpu_ctx* ctx, FrameSlot* s, const float* image0);
cudaError_t ensureRecordPool(lsdgpu_ctx* ctx);              // records.cu: the context's stream-ordered pool of device memory
cudaError_t freeRecord(lsdgpu_ctx* ctx, const FrameSlot& m); // records.cu: returns a minimized frame's blocks to their pools
cudaError_t trackPersistentSetup(lsdgpu_ctx* ctx);          // tracking.cu: launch shape of the persistent tracker
void cloudRelease(lsdgpu_ctx* ctx);                         // output.cu: frees the point-cloud reservation

// ---- device helpers shared by all kernels --------------------------------------------------------------
// util/settings.h:34-35.  UNZERO mixes float and double literals; every use converts back to float.
__device__ __forceinline__ float unzero_f(float val)
{
    double r = (val < 0 ? (val > -1e-10 ? -1e-10 : (double)val) : (val < 1e-10 ? 1e-10 : (double)val));
    return (float)r;
}

// util/globalFuncs.h:43-61 -- weights formed and summed in the reference's order (br, bl, tr, tl)
__device__ __forceinline__ float interpF(const float* __restrict__ mat, float x, float y, int width)
{
    int ix = (int)x, iy = (int)y;
    float dx = x - ix, dy = y - iy;
    float dxdy = dx * dy;
    const float* bp = mat + ix + iy * width;
    return dxdy * __ldg(bp + 1 + width) + (dy - dxdy) * __ldg(bp + width) + (dx - dxdy) * __ldg(bp + 1) + (1 - dx - dy + dxdy) * __ldg(bp);
}

// Frame::buildIDepthAndIDepthVar: one coarser idepth / idepthVar pixel from its four finer ones (frame.cuh, depth.cuh)
__device__ __forceinline__ float2 mergeIdepth4(float2 a, float2 b, float2 c, float2 d)
{   // Frame.cpp:819-871, sources visited in the order idx, idx+1, idx+sw, idx+sw+1; .x = idepth, .y = var
    float idepthSumsSum = 0, ivarSumsSum = 0;
    int num = 0;
    float2 s[4] = { a, b, c, d };
#pragma unroll
    for (int k = 0; k < 4; k++) {
        float var = s[k].y;
        if (var > 0) {
            float ivar = 1.0f / var;
            ivarSumsSum += ivar;
            idepthSumsSum += ivar * s[k].x;
            num++;
        }
    }
    if (num > 0) {
        float depth = ivarSumsSum / idepthSumsSum;
        return make_float2(1.0f / depth, num / ivarSumsSum);
    }
    return make_float2(-1.f, -1.f);
}

// Frame::prepareForStereoWith, DataStructures/Frame.cpp:295-317 (host, double -> float like the reference)
static inline void prepareStereoConsts(const float K[9], const double q[4], const double t[3], const double s, RefConst& rc)
{
    double qi[4] = { -q[0], -q[1], -q[2], q[3] };
    const double si = 1.0 / s;
    double nt[3] = { t[0] * -1.0, t[1] * -1.0, t[2] * -1.0 }, rt[3];
    lsd::quatRotate(qi, nt, rt);
    const double oTt[3] = { si * rt[0], si * rt[1], si * rt[2] };      // otherToThis.translation()
    double Ri[9], R[9];
    lsd::quatToMatrix(qi, Ri);
    lsd::quatToMatrix(q, R);
    float Rif[9];
    for (int i = 0; i < 9; i++) Rif[i] = (float)Ri[i];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            float kr = (K[i * 3 + 0] * Rif[0 * 3 + j] + K[i * 3 + 1] * Rif[1 * 3 + j]) + K[i * 3 + 2] * Rif[2 * 3 + j];
            rc.K_otherToThis_R[i * 3 + j] = kr * (float)si;
        }
    for (int i = 0; i < 3; i++) rc.otherToThis_t[i] = (float)oTt[i];
    for (int i = 0; i < 3; i++)
        rc.K_otherToThis_t[i] = (K[i * 3 + 0] * rc.otherToThis_t[0] + K[i * 3 + 1] * rc.otherToThis_t[1]) + K[i * 3 + 2] * rc.otherToThis_t[2];
    for (int i = 0; i < 3; i++) rc.thisToOther_t[i] = (float)t[i];
    float tR[9];
    for (int i = 0; i < 9; i++) tR[i] = (float)R[i] * (float)s;       // thisToOther_R
    for (int i = 0; i < 3; i++) { rc.row0[i] = tR[i * 3 + 0]; rc.row1[i] = tR[i * 3 + 1]; rc.row2[i] = tR[i * 3 + 2]; }
}
