// batches.cu -- batched tracking entry points of the C ABI (include/lsdgpu.h): permaRef overlap and tracking over a list of
// keyframe candidates (perma.cuh), and Sim3 tracking over a list of (keyframe, frame) pairs (sim3.cuh).
#include "internal.cuh"
#include "perma.cuh"
#include "sim3.cuh"

#include <stdlib.h>

// ------------------------------------------------------------------------------------------------------
// permaRef tracking (SURVEY 8f row 2)
// ------------------------------------------------------------------------------------------------------
extern "C" int lsdgpu_frame_set_perma_ref(lsdgpu_ctx* ctx, int kf_id, int* num_points_out)
{ LSD_LOCK(ctx);   // Frame::setPermaRef -> reference->makePointCloud(QUICK_KF_CHECK_LVL) + copy (Frame.cpp:149-174, TrackingReference.cpp:96-147)
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return failMissing(ctx, kf_id, "unknown keyframe id");
    int r = ensureIdepthPyramid(ctx, kf);
    if (r) return r;
    const LevelCam& c = ctx->cam[QUICK_KF_CHECK_LVL];
    const int w = c.w, h = c.h, n = w * h;
    std::vector<float> id(n), var(n), col(n);
    LSD_CHECK(ctx, cudaMemcpyAsync(id.data(), kf->idepth[QUICK_KF_CHECK_LVL], n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaMemcpyAsync(var.data(), kf->idepthVar[QUICK_KF_CHECK_LVL], n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaMemcpyAsync(col.data(), kf->image[QUICK_KF_CHECK_LVL], n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    std::vector<float4> pc;
    std::vector<float> pv;
    for (int x = 1; x < w - 1; x++)                    // x outer, y inner: the reference's point order (:128-129)
        for (int y = 1; y < h - 1; y++) {
            const int idx = x + y * w;
            if (var[idx] <= 0 || id[idx] == 0) continue;
            const float sc = 1.0f / id[idx];
            pc.push_back(make_float4(sc * (c.fxi * x + c.cxi), sc * (c.fyi * y + c.cyi), sc * 1, col[idx]));
            pv.push_back(var[idx]);
        }
    kf->permaNumPts = (int)pc.size();
    if (kf->permaNumPts) {
        LSD_CHECK(ctx, cudaMemcpyAsync(kf->permaPC, pc.data(), pc.size() * 16, cudaMemcpyHostToDevice, ctx->stream));
        LSD_CHECK(ctx, cudaMemcpyAsync(kf->permaVar, pv.data(), pv.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
        LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (num_points_out) *num_points_out = kf->permaNumPts;
    return 0;
}

static int fillPermaItems(lsdgpu_ctx* ctx, int n, const int* kf_ids, const double* qt, std::vector<PermaItem>& items)
{
    if (n <= 0 || n > LSD_MAX_PERMA_BATCH) return lsd_fail(ctx, "bad candidate count");
    items.resize(n);
    for (int i = 0; i < n; i++) {
        FrameSlot* kf = findFrame(ctx, kf_ids[i]);           // a minimized keyframe's permaRef is read from its record
        if (!kf) return lsd_fail(ctx, "unknown keyframe id");
        if (kf->permaNumPts <= 0) return lsd_fail(ctx, "keyframe has no permaRef (call lsdgpu_frame_set_perma_ref)");
        lsd::SE3<double> T;
        for (int k = 0; k < 4; k++) T.q[k] = qt[7 * i + k];
        for (int k = 0; k < 3; k++) T.t[k] = qt[7 * i + 4 + k];
        const lsd::SE3<float> Tf = lsd::se3Cast<float>(T);                 // referenceToFrameOrg.cast<float>(), :125,168
        items[i].pc = kf->permaPC; items[i].var = kf->permaVar; items[i].n = kf->permaNumPts;
        for (int k = 0; k < 4; k++) items[i].refToFrame[k] = Tf.q[k];
        for (int k = 0; k < 3; k++) items[i].refToFrame[4 + k] = Tf.t[k];
    }
    LSD_CHECK(ctx, cudaMemcpyAsync(ctx->dPermaItems, items.data(), n * sizeof(PermaItem), cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

extern "C" int lsdgpu_perma_overlap_batch(lsdgpu_ctx* ctx, int n, const int* kf_ids, const double* refToFrame_qt, float* usage_out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    std::vector<PermaItem> items;
    int r = fillPermaItems(ctx, n, kf_ids, refToFrame_qt, items);
    if (r) return r;
    const LevelCam& c = ctx->cam[QUICK_KF_CHECK_LVL];
    float* dUsage = (float*)ctx->dPermaResults;
    k_perma_overlap<<<n, 128, 0, ctx->stream>>>((const PermaItem*)ctx->dPermaItems, c.fx, c.fy, c.cx, c.cy, c.w - 1, c.h - 1, dUsage);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    LSD_CHECK(ctx, cudaMemcpyAsync(usage_out, dUsage, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int lsdgpu_perma_track_batch(lsdgpu_ctx* ctx, int n, const int* kf_ids, int frame_id, const double* refToFrame_init_qt,
                                        lsdgpu_track_result* results)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* fr = findSlot(ctx, frame_id);
    if (!fr) return failMissing(ctx, frame_id, "unknown frame id");
    std::vector<PermaItem> items;
    int r = fillPermaItems(ctx, n, kf_ids, refToFrame_init_qt, items);
    if (r) return r;
    TrackParams P;
    memset(&P, 0, sizeof(P));
    const LevelCam& c = ctx->cam[QUICK_KF_CHECK_LVL];
    TrackLevelParams& L = P.lvl[QUICK_KF_CHECK_LVL];
    L.frameGrad = fr->grad[QUICK_KF_CHECK_LVL];
    L.w = c.w; L.h = c.h; L.fx = c.fx; L.fy = c.fy; L.cx = c.cx; L.cy = c.cy;
    L.fxi = c.fxi; L.fyi = c.fyi; L.cxi = c.cxi; L.cyi = c.cyi;
    P.W = ctx->w; P.H = ctx->h;
    lsdgpu_track_settings st;
    lsdgpu_default_track_settings(&st);
    // TestTrack settings (util/settings.h:379-382) mapped onto level 4
    st.lambdaInitial[QUICK_KF_CHECK_LVL] = 0; st.stepSizeMin[QUICK_KF_CHECK_LVL] = 1e-3f;
    st.convergenceEps[QUICK_KF_CHECK_LVL] = 0.98f; st.maxItsPerLvl[QUICK_KF_CHECK_LVL] = 5;
    P.st = st;
    P.C.cameraPixelNoise2 = ctx->g.cameraPixelNoise2; P.C.var_weight = st.var_weight; P.C.huber_half = st.huber_d / 2;
    P.useAffine = ctx->g.useAffineLightningEstimation;
    P.minLevel = QUICK_KF_CHECK_LVL;
    P.kmax = 1;                                   // one pose per pass: the candidates are independent CTAs already
    PermaResult* dRes = (PermaResult*)ctx->dPermaResults;
    k_perma_track<<<n, PERMA_THREADS, 0, ctx->stream>>>(P, (const PermaItem*)ctx->dPermaItems, dRes);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    std::vector<PermaResult> hres(n);
    LSD_CHECK(ctx, cudaMemcpyAsync(hres.data(), dRes, n * sizeof(PermaResult), cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < n; i++) {
        lsdgpu_track_result& o = results[i];
        memset(&o, 0, sizeof(o));
        const PermaResult& h = hres[i];
        o.pointUsage = h.pointUsage; o.lastGoodCount = h.goodCount; o.lastBadCount = h.badCount; o.lastMeanRes = h.meanRes;
        o.affineEstimation_a = h.affine_a; o.affineEstimation_b = h.affine_b;
        o.numCalcResidualCalls[QUICK_KF_CHECK_LVL] = h.nRes; o.numCalcWarpUpdateCalls[QUICK_KF_CHECK_LVL] = h.nUpd;
        if (h.diverged) { o.frameToRef_qt[3] = 1; o.diverged = 1; continue; }             // return SE3(), :180-185
        o.lastResidual = h.lastResidual;                                                // :265
        o.trackingWasGood = h.goodCount / (c.w * c.h) > 0.04f && h.goodCount / (h.goodCount + h.badCount) > 0.5f;   // :267-269
        lsd::SE3<float> T;
        for (int k = 0; k < 4; k++) T.q[k] = h.refToFrame[k];
        for (int k = 0; k < 3; k++) T.t[k] = h.refToFrame[4 + k];
        const lsd::SE3<double> Td = lsd::se3Cast<double>(T);                            // toSophus(referenceToFrame), :271
        for (int k = 0; k < 4; k++) o.frameToRef_qt[k] = Td.q[k];
        for (int k = 0; k < 3; k++) o.frameToRef_qt[4 + k] = Td.t[k];
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------------
// Sim3 tracking, batched (SURVEY 8f row 1)
// ------------------------------------------------------------------------------------------------------
static int sim3Launch(lsdgpu_ctx* ctx, int n, const int* ref_ids, const int* frame_ids, const double* qts, bool qtsIsRefToFrame,
                      int startLevel, int finalLevel, const lsdgpu_track_settings* s, int evalOnly, float evalA, float evalB,
                      std::vector<Sim3Out>& hout)
{
    if (n <= 0 || n > S3_MAX_BATCH) return lsd_fail(ctx, "bad problem count");
    if (startLevel < 0 || startLevel >= LSD_LEVELS || finalLevel < 0 || finalLevel > startLevel) return lsd_fail(ctx, "bad level range");
    std::vector<Sim3Item> items(n);
    for (int i = 0; i < n; i++) {
        FrameSlot* kf = findSlot(ctx, ref_ids[i]);
        FrameSlot* fr = findSlot(ctx, frame_ids[i]);
        if (!kf || !fr) return failMissing(ctx, kf ? frame_ids[i] : ref_ids[i], "unknown frame id");
        int r = ensureIdepthPyramid(ctx, kf);       // reference->makePointCloud(lvl), Sim3Tracker.cpp:174
        if (r) return r;
        r = ensureIdepthPyramid(ctx, fr);           // frame->idepth(level) / idepthVar(level), :467-468
        if (r) return r;
        for (int l = 0; l < LSD_LEVELS; l++) {
            items[i].kfIdepth[l] = kf->idepth[l]; items[i].kfVar[l] = kf->idepthVar[l]; items[i].kfGrad[l] = kf->grad[l];
            items[i].frGrad[l] = fr->grad[l]; items[i].frIdepth[l] = fr->idepth[l]; items[i].frVar[l] = fr->idepthVar[l];
        }
        lsd::Sim3 T = lsd::sim3FromQts(qts + 8 * i);
        if (!qtsIsRefToFrame) T = lsd::sim3Inverse(T);                  // :161
        for (int k = 0; k < 4; k++) items[i].refToFrame[k] = T.q[k];
        for (int k = 0; k < 3; k++) items[i].refToFrame[4 + k] = T.t[k];
    }
    LSD_CHECK(ctx, cudaMemcpyAsync(ctx->dSim3Items, items.data(), n * sizeof(Sim3Item), cudaMemcpyHostToDevice, ctx->stream));
    Sim3Params P;
    memset(&P, 0, sizeof(P));
    for (int l = 0; l < LSD_LEVELS; l++) {
        const LevelCam& c = ctx->cam[l];
        Sim3Level& L = P.lvl[l];
        L.w = c.w; L.h = c.h; L.fx = c.fx; L.fy = c.fy; L.cx = c.cx; L.cy = c.cy; L.fxi = c.fxi; L.fyi = c.fyi; L.cxi = c.cxi; L.cyi = c.cyi;
    }
    lsdgpu_track_settings ds;
    if (!s) { lsdgpu_default_track_settings(&ds); s = &ds; }
    P.st = *s;
    P.cameraPixelNoise2 = ctx->g.cameraPixelNoise2;
    P.useAffine = ctx->g.useAffineLightningEstimation;
    P.W = ctx->w; P.H = ctx->h;
    P.startLevel = startLevel; P.finalLevel = finalLevel;
    P.evalOnly = evalOnly; P.evalA = evalA; P.evalB = evalB;
    // one cluster per problem: 8 CTAs (the portable maximum) unless the batch alone fills the GPU
    int cs = 8;
    if (const char* e = getenv("LSDGPU_SIM3_CLUSTER")) cs = atoi(e);
    else if (n >= 2 * ctx->smCount) cs = 1;
    else if (n * 8 > 2 * ctx->smCount) cs = (n * 4 > 2 * ctx->smCount) ? ((n * 2 > 2 * ctx->smCount) ? 1 : 2) : 4;
    if (cs != 1 && cs != 2 && cs != 4 && cs != 8) cs = 8;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(n * cs); cfg.blockDim = dim3(S3_THREADS); cfg.dynamicSmemBytes = 0; cfg.stream = ctx->stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    LSD_CHECK(ctx, cudaLaunchKernelEx(&cfg, k_sim3_track, P, (const Sim3Item*)ctx->dSim3Items, (Sim3Out*)ctx->dSim3Outs));
    LAUNCH(ctx);
    hout.resize(n);
    LSD_CHECK(ctx, cudaMemcpyAsync(hout.data(), ctx->dSim3Outs, n * sizeof(Sim3Out), cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    if (getenv("LSDGPU_SIM3_DEBUG")) {
        const Sim3Out& o = hout[0];
        int ev = 0;
        for (int l = 0; l < LSD_LEVELS; l++) ev += o.nRes[l];
        fprintf(stderr, "[sim3] cluster=%d evals=%d cycles: points=%lld ctaReduce=%lld exchange=%lld serialLM=%lld\n", cs, ev, o.cyc[0], o.cyc[1], o.cyc[2], o.cyc[3]);
    }
    return 0;
}

extern "C" int lsdgpu_sim3_eval(lsdgpu_ctx* ctx, int ref_kf_id, int frame_id, int level, const double refToFrame_qts[8],
                                float affine_a, float affine_b, const lsdgpu_track_settings* s, lsdgpu_sim3_eval_result* out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    std::vector<Sim3Out> h;
    int r = sim3Launch(ctx, 1, &ref_kf_id, &frame_id, refToFrame_qts, true, level, level, s, 1, affine_a, affine_b, h);
    if (r) return r;
    const float* sm = h[0].sums;
    sim3AssembleLGS7(sm, out->A, out->b);
    const Sim3Res res = sim3Finish(sm);
    out->num_constraints = 2 * res.warpedSize;
    out->sumResD = sm[S3_RESD]; out->sumResP = sm[S3_RESP]; out->numTermsD = (int)sm[S3_NUMD]; out->numTermsP = (int)sm[S3_NUMP];
    out->mean = res.mean; out->meanD = res.meanD; out->meanP = res.meanP;
    out->warpedSize = res.warpedSize; out->pointUsage = res.pointUsage;
    out->affine_a_lastIt = res.a_lastIt; out->affine_b_lastIt = res.b_lastIt;
    return 0;
}

extern "C" int lsdgpu_sim3_track_batch(lsdgpu_ctx* ctx, int n, const int* ref_kf_ids, const int* frame_ids, const double* frameToRef_init_qts,
                                       int start_level, int final_level, const lsdgpu_track_settings* s, lsdgpu_sim3_result* results)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    std::vector<Sim3Out> h;
    int r = sim3Launch(ctx, n, ref_kf_ids, frame_ids, frameToRef_init_qts, false, start_level, final_level, s, 0, 1.f, 0.f, h);
    if (r) return r;
    for (int i = 0; i < n; i++) {
        lsdgpu_sim3_result& o = results[i];
        const Sim3Out& d = h[i];
        memset(&o, 0, sizeof(o));
        o.frameToRef_qts[3] = 1; o.frameToRef_qts[7] = 1;                               // Sim3()
        o.pointUsage = d.pointUsage; o.affineEstimation_a = d.affine_a; o.affineEstimation_b = d.affine_b;
        for (int l = 0; l < LSD_LEVELS; l++) { o.numCalcResidualCalls[l] = d.nRes[l]; o.numCalcWarpUpdateCalls[l] = d.nUpd[l]; }
        if (d.early) { o.diverged = (d.early == 1); continue; }                         // :184-187, :212-217, :231-235
        float b7[7];
        sim3AssembleLGS7(d.lgs, o.lastSim3Hessian, b7);                                 // lastSim3Hessian = ls7.A, :360
        lsd::Sim3 T;
        for (int k = 0; k < 4; k++) T.q[k] = d.refToFrame[k];
        for (int k = 0; k < 3; k++) T.t[k] = d.refToFrame[4 + k];
        if (lsd::sim3Scale(T) <= 0) { o.diverged = 1; continue; }                       // :363-367
        o.lastResidual = d.resMean; o.lastDepthResidual = d.resMeanD; o.lastPhotometricResidual = d.resMeanP;   // :369-371
        lsd::sim3ToQts(lsd::sim3Inverse(T), o.frameToRef_qts);                          // :374
    }
    return 0;
}

extern "C" int lsdgpu_sim3_track(lsdgpu_ctx* ctx, int ref_kf_id, int frame_id, const double frameToRef_init_qts[8],
                                 int start_level, int final_level, const lsdgpu_track_settings* s, lsdgpu_sim3_result* out)
{ LSD_LOCK(ctx);
    return lsdgpu_sim3_track_batch(ctx, 1, &ref_kf_id, &frame_id, frameToRef_init_qts, start_level, final_level, s, out);
}
