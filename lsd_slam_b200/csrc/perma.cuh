// perma.cuh -- batched permaRef tracking (SURVEY 8f row 2: the first "next" row after the hot path).
//
// Replaces (paths relative to lsd_slam_core/src/):
//   Frame::setPermaRef                   DataStructures/Frame.cpp:149-174   (snapshot of the keyframe's level-4 point cloud)
//   SE3Tracker::checkPermaRefOverlap     Tracking/SE3Tracker.cpp:121-157
//   SE3Tracker::trackFrameOnPermaref     Tracking/SE3Tracker.cpp:162-272
// Callers in the reference evaluate MANY keyframe candidates against one frame, one call after the other
// (Relocalizer.cpp:172,188; TrackableKeyFrameSearch.cpp:126,135; SlamSystem.cpp:1298,1304).  Here a whole candidate list
// is one launch: one CTA per candidate runs the complete level-4 LM loop on its own (the problems are independent, so
// there is no grid barrier and no exchange at all) with the same evalPoint() / lmAdvance() as the main tracker (one pose per pass: kmax = 1).
#pragma once
#include "track_common.cuh"

#define QUICK_KF_CHECK_LVL 4            // util/settings.h:104
#define PERMA_THREADS 256

// checkPermaRefOverlap for a list of candidates: CTA b -> usage[b]
__global__ void __launch_bounds__(128) k_perma_overlap(const PermaItem* __restrict__ items, float fx_l, float fy_l, float cx_l, float cy_l,
                                                       int w2, int h2, float* __restrict__ usage)
{
    __shared__ float sm[4];
    const PermaItem it = items[blockIdx.x];
    lsd::SE3<float> T;
    for (int i = 0; i < 4; i++) T.q[i] = it.refToFrame[i];
    for (int i = 0; i < 3; i++) T.t[i] = it.refToFrame[4 + i];
    float R[9];
    lsd::quatToMatrix(T.q, R);
    float s = 0.f;
    for (int k = threadIdx.x; k < it.n; k += blockDim.x) {
        const float4 p = __ldg(it.pc + k);
        const float Wx = ((R[0] * p.x + R[1] * p.y) + R[2] * p.z) + T.t[0];
        const float Wy = ((R[3] * p.x + R[4] * p.y) + R[5] * p.z) + T.t[1];
        const float Wz = ((R[6] * p.x + R[7] * p.y) + R[8] * p.z) + T.t[2];
        const float u_new = (Wx / Wz) * fx_l + cx_l;
        const float v_new = (Wy / Wz) * fy_l + cy_l;
        if ((u_new > 0 && v_new > 0 && u_new < w2 && v_new < h2)) {             // SE3Tracker.cpp:148
            const float depthChange = p.z / Wz;
            s += depthChange < 1 ? depthChange : 1;
        }
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) usage[blockIdx.x] = ((sm[0] + sm[1]) + (sm[2] + sm[3])) / (float)it.n;     // :155
}

// trackFrameOnPermaref for a list of candidates: CTA b runs the whole LM loop of candidate b.
// p carries the shared part (level-4 intrinsics and gradient image of the frame, TestTrack settings mapped onto level 4).
__global__ void __launch_bounds__(PERMA_THREADS) k_perma_track(const __grid_constant__ TrackParams p, const PermaItem* __restrict__ items,
                                                               PermaResult* __restrict__ results)
{
    __shared__ alignas(LMShared) unsigned char shStorage[sizeof(LMShared)];   // raw storage: Proposal holds a type with a constructor
    LMShared& sh = *reinterpret_cast<LMShared*>(shStorage);
    __shared__ alignas(LMState) unsigned char lmStorage[sizeof(LMState)];     // every field is written before use; no constructor in shared memory
    LMState& lm = *reinterpret_cast<LMState*>(lmStorage);
    __shared__ float sm[PERMA_THREADS / 32][EV_NCH];
    const PermaItem it = items[blockIdx.x];
    const TrackLevelParams& L = p.lvl[QUICK_KF_CHECK_LVL];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 4; i++) lm.refToFrame.q[i] = it.refToFrame[i];
        for (int i = 0; i < 3; i++) lm.refToFrame.t[i] = it.refToFrame[4 + i];
        for (int l = 0; l < LSD_LEVELS; l++) { lm.nRes[l] = 0; lm.nUpd[l] = 0; lm.nEval[l] = 0; lm.nPts[l] = 0.f; }
        lm.chainBase = 0; lm.statsFrom = 0; lm.commitLast = 0; lm.posesEvaluated = 0;
        lm.affine_a = 1.f; lm.affine_b = 0.f; lm.lastErr = 0.f; lm.last_residual = 0.f; lm.LM_lambda = 0.f;
        lm.diverged = 0; lm.incTry = 0; lm.iteration = 0; lm.dbg[0] = lm.dbg[1] = lm.dbg[2] = lm.dbg[3] = 0;
        lm.lvl = QUICK_KF_CHECK_LVL; lm.phase = PH_INIT;
        sh.lvl = lm.lvl; sh.action = ACT_CONTINUE; sh.nPose = 1;
        setEvalPose(sh.pose[0], lm.refToFrame, lm.affine_a, lm.affine_b);
    }
    __syncthreads();
    const float4* fg = L.frameGrad;
    const int w = L.w, h = L.h;
    while (true) {
        const EvalPose P = sh.pose[0];      // p.kmax == 1: one pose per pass
        PointAcc acc;
#pragma unroll
        for (int c = 0; c < EV_NCH; c++) acc.v[c] = 0.f;
        for (int k = threadIdx.x; k < it.n; k += PERMA_THREADS) {
            const float4 pt = __ldg(it.pc + k);
            auto tap = [fg, w](float u, float v, float& o0, float& o1, float& o2) { interp43(fg, u, v, w, o0, o1, o2); };
            evalPoint(pt.x, pt.y, pt.z, pt.w, __ldg(it.var + k), P, p.C, L.fx, L.fy, L.cx, L.cy, w, h, tap, acc);   // idxBuf == 0: no mask (:179)
        }
        __syncthreads();
        warpReduceAcc(acc, lane, sm[warp]);
        __syncthreads();
        if (threadIdx.x < EV_NCH) {
            float s = 0.f;
#pragma unroll
            for (int wi = 0; wi < PERMA_THREADS / 32; wi++) s += sm[wi][threadIdx.x];
            sh.sums[threadIdx.x] = s;
        }
        __syncthreads();
        if (threadIdx.x < 32) lmAdvance(p, lm, sh, threadIdx.x);        // warp 0: decisions on lane 0, the solve in buildChain
        __syncthreads();
        if (sh.action != ACT_CONTINUE) break;
    }
    if (threadIdx.x == 0) {
        PermaResult& r = results[blockIdx.x];
        lsdgpu_eval_result ev;
        evalFinish(sh.sums, &ev);
        for (int i = 0; i < 4; i++) r.refToFrame[i] = lm.refToFrame.q[i];
        for (int i = 0; i < 3; i++) r.refToFrame[4 + i] = lm.refToFrame.t[i];
        r.pointUsage = ev.pointUsage; r.goodCount = ev.goodCount; r.badCount = ev.badCount; r.meanRes = ev.meanRes;
        r.lastResidual = lm.lastErr;                                    // lastResidual = lastErr, SE3Tracker.cpp:265
        r.affine_a = lm.affine_a; r.affine_b = lm.affine_b;
        r.diverged = lm.diverged;
        r.nRes = lm.nRes[QUICK_KF_CHECK_LVL]; r.nUpd = lm.nUpd[QUICK_KF_CHECK_LVL];
    }
}
