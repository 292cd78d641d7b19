// sim3.cuh -- Sim3Tracker::trackFrameSim3 on the device, batched over independent (reference keyframe, frame) pairs
// (SURVEY 8f row 1).
//
// Replaces (paths relative to lsd_slam_core/src/):
//   Sim3Tracker::trackFrameSim3               Tracking/Sim3Tracker.cpp:149-382   (LM schedule, early returns, final warp update)
//   Sim3Tracker::calcSim3Buffers              Tracking/Sim3Tracker.cpp:414-607   (warp, ESM gradient, photometric + depth residual)
//   Sim3Tracker::calcSim3WeightsAndResidual   Tracking/Sim3Tracker.cpp:748-856
//   Sim3Tracker::calcSim3LGS                  Tracking/Sim3Tracker.cpp:992-1047
//   LGS4 / LGS6 / LGS7::initializeFrom        Tracking/LGSX.h:45-176, 184-402, 411-443
//   TrackingReference::makePointCloud         Tracking/TrackingReference.cpp:96-147  (never materialised, as in track.cuh)
// Callers (SlamSystem::tryTrackSim3, SlamSystem.cpp:1043-1127; testConstraint :1130-1174) run two trackings per candidate and
// several candidates per new keyframe, all independent: here a whole list is ONE launch.  One thread-block CLUSTER per
// problem runs the complete coarse-to-fine LM loop on its own: the CTAs of a cluster split the pixels of the level, exchange
// their S3_NCH partial sums through distributed shared memory behind one hardware cluster barrier per evaluation, and every
// CTA then takes the (identical, deterministic) LM decision redundantly -- 7x7 LDL^T and the Sim3 exp/multiply in double
// on thread 0 -- so there is no grid barrier, no global-memory exchange and no host round trip inside a tracking.
#pragma once
#include <cooperative_groups.h>
#include "track_common.cuh"

namespace cg = cooperative_groups;

#define S3_THREADS 512

struct Sim3Level {
    int w, h;
    float fx, fy, cx, cy, fxi, fyi, cxi, cyi;
};
struct Sim3Params {
    Sim3Level lvl[LSD_LEVELS];
    lsdgpu_track_settings st;
    float cameraPixelNoise2;
    int useAffine;
    int W, H;                           // tracker construction size (the "too few points" test, Sim3Tracker.cpp:182)
    int startLevel, finalLevel;
    int evalOnly;                       // 1: one evaluation at level startLevel with the given pose / affine (parity hook)
    float evalA, evalB;
};

struct Sim3Pose {
    float R[9], t[3], roll[4];          // rxso3 matrix, translation, xRoll0 xRoll1 yRoll0 yRoll1
    float a, b;
};

// One reference pixel -> all channels.  Sim3Tracker.cpp:472-585 (buffers), :762-835 (weights), :1001-1038 (LGS).
__device__ __forceinline__ void sim3EvalPoint(float px, float py, float pz, float refGx, float refGy, float color, float var,
                                              const Sim3Pose& P, const Sim3Level& L, const float4* __restrict__ frGrad,
                                              const float* __restrict__ frIdepth, const float* __restrict__ frVar,
                                              float var_weight, float huber_d, float cameraPixelNoise2, float* acc)
{
    const float Wx = ((P.R[0] * px + P.R[1] * py) + P.R[2] * pz) + P.t[0];
    const float Wy = ((P.R[3] * px + P.R[4] * py) + P.R[5] * pz) + P.t[1];
    const float Wz = ((P.R[6] * px + P.R[7] * py) + P.R[8] * pz) + P.t[2];
    const float u_new = (Wx / Wz) * L.fx + L.cx;
    const float v_new = (Wy / Wz) * L.fy + L.cy;
    acc[S3_REFNUM] += 1.f;
    if (!(u_new > 1 && v_new > 1 && u_new < L.w - 2 && v_new < L.h - 2)) return;          // :482-483

    float r0, r1, r2;
    interp43(frGrad, u_new, v_new, L.w, r0, r1, r2);
    const float rotatedGradX = P.roll[0] * refGx + P.roll[1] * refGy;                      // :499-500
    const float rotatedGradY = P.roll[2] * refGx + P.roll[3] * refGy;
    const float gx = L.fx * 0.5f * (r0 + rotatedGradX);                                   // :502-503
    const float gy = L.fy * 0.5f * (r1 + rotatedGradY);

    const float c1 = P.a * color + P.b;                                                   // :510-520
    const float c2 = r2;
    const float rp = c1 - c2;
    const float weight = fabsf(rp) < 2.0f ? 1 : 2.0f / fabsf(rp);
    acc[S3_SXX] += c1 * c1 * weight;
    acc[S3_SYY] += c2 * c2 * weight;
    acc[S3_SX] += c1 * weight;
    acc[S3_SY] += c2 * weight;
    acc[S3_SW] += weight;

    const int idx_rounded = (int)(u_new + 0.5f) + L.w * (int)(v_new + 0.5f);               // :527-542
    const float var_frameDepth = __ldg(frVar + idx_rounded);
    const float ref_idepth = 1.0f / Wz;
    const float d = 1.0f / pz;
    float rd, wiv;
    if (var_frameDepth > 0) { rd = ref_idepth - __ldg(frIdepth + idx_rounded); wiv = var_frameDepth; }
    else { rd = -1; wiv = -1; }
    const float depthChange = pz / Wz;                                                    // :583-584
    acc[S3_USAGE] += depthChange < 1 ? depthChange : 1;

    // calcSim3WeightsAndResidual
    const float s = var_weight * var;
    const float sv = var_weight * wiv;
    const float g0 = (P.t[0] * Wz - P.t[2] * Wx) / (Wz * Wz * d);
    const float g1 = (P.t[1] * Wz - P.t[2] * Wy) / (Wz * Wz * d);
    const float g2 = (Wz - P.t[2]) / (Wz * Wz * d);
    const float drpdd = gx * g0 + gy * g1;
    const float w_p = 1.0f / (cameraPixelNoise2 + s * drpdd * drpdd);
    const float w_d = 1.0f / (sv + g2 * g2 * s);
    const float weighted_rd = fabsf(rd * sqrtf(w_d));
    const float weighted_rp = fabsf(rp * sqrtf(w_p));
    const float weighted_abs_res = sv > 0 ? weighted_rd + weighted_rp : weighted_rp;
    const float wh = fabsf(weighted_abs_res < huber_d ? 1 : huber_d / weighted_abs_res);
    float wd = 0.f;
    if (sv > 0) {
        acc[S3_RESD] += wh * w_d * rd * rd;
        acc[S3_NUMD] += 1.f;
        wd = wh * w_d;
    }
    acc[S3_RESP] += wh * w_p * rp * rp;
    acc[S3_NUMP] += 1.f;
    const float wp = wh * w_p;

    // calcSim3LGS (rows 3 and 4 carry double literals in the reference)
    const float z = 1.0f / Wz;
    const float z_sqr = 1.0f / (Wz * Wz);
    float v[6], v4[4];
    v[0] = z * gx + 0;
    v[1] = 0 + z * gy;
    v[2] = (-Wx * z_sqr) * gx + (-Wy * z_sqr) * gy;
    v[3] = (float)((double)((-Wx * Wy * z_sqr) * gx) + (-(1.0 + (double)(Wy * Wy * z_sqr))) * (double)gy);
    v[4] = (float)((1.0 + (double)(Wx * Wx * z_sqr)) * (double)gx + (double)((Wx * Wy * z_sqr) * gy));
    v[5] = (-Wy * z) * gx + (Wx * z) * gy;
    v4[0] = z_sqr;
    v4[1] = z_sqr * Wy;
    v4[2] = -z_sqr * Wx;
    v4[3] = z;
    // LGS6::update / LGS4::update in the association order of the reference's SSE path (J_i w first, LGSX.h:139-160,
    // 337-386), one fused multiply-add per channel: this part of the kernel is issue-bound, and tracking parity is
    // tolerance-based (the CPU paths of the reference differ among themselves by the same re-association)
    float vw[6], v4w[4];
#pragma unroll
    for (int i = 0; i < 6; i++) vw[i] = v[i] * wp;
#pragma unroll
    for (int i = 0; i < 4; i++) v4w[i] = v4[i] * wd;
    int k = 0;
#pragma unroll
    for (int i = 0; i < 6; i++)
#pragma unroll
        for (int j = i; j < 6; j++) { acc[S3_A6 + k] = fmaf(vw[i], v[j], acc[S3_A6 + k]); k++; }
#pragma unroll
    for (int i = 0; i < 6; i++) acc[S3_B6 + i] = fmaf(vw[i], rp, acc[S3_B6 + i]);
    k = 0;
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = i; j < 4; j++) { acc[S3_A4 + k] = fmaf(v4w[i], v4[j], acc[S3_A4 + k]); k++; }
#pragma unroll
    for (int i = 0; i < 4; i++) acc[S3_B4 + i] = fmaf(v4w[i], rd, acc[S3_B4 + i]);
}

// ---- interpretation of the sums (host and device) ---------------------------------------------------------------
struct Sim3Res { float mean, meanD, meanP; int warpedSize; float pointUsage, a_lastIt, b_lastIt; };
LSD_HD Sim3Res sim3Finish(const float* s)
{
    Sim3Res r;
    r.mean = (s[S3_RESD] + s[S3_RESP]) / (float)((int)s[S3_NUMD] + (int)s[S3_NUMP]);    // :838-840
    r.meanD = s[S3_RESD] / (float)(int)s[S3_NUMD];
    r.meanP = s[S3_RESP] / (float)(int)s[S3_NUMP];
    r.warpedSize = (int)s[S3_NUMP];
    r.pointUsage = s[S3_USAGE] / s[S3_REFNUM];                                             // :589
    const float sxx = s[S3_SXX], syy = s[S3_SYY], sx = s[S3_SX], sy = s[S3_SY], sw = s[S3_SW];
    r.a_lastIt = sqrtf((syy - sy * sy / sw) / (sxx - sx * sx / sw));                       // :591-592
    r.b_lastIt = (sy - r.a_lastIt * sx) / sw;
    return r;
}
// LGS7::initializeFrom(ls6, ls4), LGSX.h:422-441; A7/b7 undivided (b carries the reference's minus sign)
LSD_HD void sim3AssembleLGS7(const float* lgs, float A7[49], float b7[7])
{
    for (int i = 0; i < 49; i++) A7[i] = 0.f;
    for (int i = 0; i < 7; i++) b7[i] = 0.f;
    int k = 0;
    for (int i = 0; i < 6; i++)
        for (int j = i; j < 6; j++) { A7[i * 7 + j] = lgs[S3_A6 + k]; A7[j * 7 + i] = lgs[S3_A6 + k]; k++; }
    for (int i = 0; i < 6; i++) b7[i] = -lgs[S3_B6 + i];
    const int remap[4] = { 2, 3, 4, 6 };
    float A4[16];
    k = 0;
    for (int i = 0; i < 4; i++)
        for (int j = i; j < 4; j++) { A4[i * 4 + j] = lgs[S3_A4 + k]; A4[j * 4 + i] = lgs[S3_A4 + k]; k++; }
    for (int i = 0; i < 4; i++) {
        b7[remap[i]] += -lgs[S3_B4 + i];
        for (int j = 0; j < 4; j++) A7[remap[i] * 7 + remap[j]] += A4[i * 4 + j];
    }
}

// ---- the LM state machine of trackFrameSim3 (thread 0 of every CTA, identical in all CTAs of a cluster) -----------
enum { S3_PH_INIT = 0, S3_PH_TRY = 1, S3_PH_FINAL = 2, S3_PH_EVALONLY = 3 };
struct Sim3LM {
    lsd::Sim3 refToFrame, cand;
    float lgs[S3_NLGS];
    float ncons;                        // ls7.num_constraints of lgs
    float lastErrMean;
    float resMean, resMeanD, resMeanP;  // finalResidual
    float affine_a, affine_b, LM_lambda, absInc, pointUsage;
    int lvl, phase, iteration, incTry, warpUpToDate, early, done;
    int nRes[LSD_LEVELS], nUpd[LSD_LEVELS];
};
struct Sim3Shared {
    Sim3Pose pose;
    int lvl, done;
};

// exp(inc) * T on the device in double, latency-trimmed for the one thread that runs it: one sincos (half angle; the
// full angle by the double-angle identities), one exp, reciprocals instead of repeated divisions, W * upsilon by cross
// products.  Same algebra as lsd::sim3Exp / sim3Mul (hostmath.h; sim3.hpp:418-428, 609-648, 257-260); agrees to ~1e-15.
__device__ __forceinline__ lsd::Sim3 sim3ExpMulFast(const float* inc, const lsd::Sim3& T)
{
    const double ux = inc[0], uy = inc[1], uz = inc[2], wx = inc[3], wy = inc[4], wz = inc[5], sigma = inc[6];
    const double scale = exp(sigma);
    const double theta_sq = wx * wx + wy * wy + wz * wz;
    double imag, real, A, B, C;
    const bool smallSigma = fabs(sigma) < 1e-10;
    C = smallSigma ? 1.0 : (scale - 1.0) / sigma;
    if (theta_sq < 1e-20) {
        const double theta_po4 = theta_sq * theta_sq;
        imag = 0.5 - (1.0 / 48.0) * theta_sq + (1.0 / 3840.0) * theta_po4;
        real = 1.0 - 0.5 * theta_sq + (1.0 / 384.0) * theta_po4;
        if (smallSigma) { A = 0.5; B = 1.0 / 6.0; }
        else {
            const double inv_s = 1.0 / sigma, inv_s2 = inv_s * inv_s;
            A = ((sigma - 1.0) * scale + 1.0) * inv_s2;
            B = ((0.5 * sigma * sigma - sigma + 1.0) * scale) * inv_s2 * inv_s;
        }
    } else {
        const double theta = sqrt(theta_sq), inv_theta = 1.0 / theta, inv_tsq = inv_theta * inv_theta;
        double sh_, ch_;
        sincos(0.5 * theta, &sh_, &ch_);
        imag = sh_ * inv_theta;
        real = ch_;
        const double sinT = 2.0 * sh_ * ch_, cosT = 1.0 - 2.0 * sh_ * sh_;
        if (smallSigma) {
            A = (1.0 - cosT) * inv_tsq;
            B = (theta - sinT) * inv_tsq * inv_theta;
        } else {
            const double sa = scale * sinT, sb = scale * cosT, inv_c = 1.0 / (theta_sq + sigma * sigma);
            A = (sa * sigma + (1.0 - sb) * theta) * inv_theta * inv_c;
            B = (C - ((sb - 1.0) * sigma + sa * theta) * inv_c) * inv_tsq;
        }
    }
    const double uq[4] = { imag * wx, imag * wy, imag * wz, real };          // unit quaternion of the increment
    // W * upsilon,  W = A Omega + B Omega^2 + C I :  Omega u = w x u
    const double k1x = wy * uz - wz * uy, k1y = wz * ux - wx * uz, k1z = wx * uy - wy * ux;
    const double k2x = wy * k1z - wz * k1y, k2y = wz * k1x - wx * k1z, k2z = wx * k1y - wy * k1x;
    const double tx = A * k1x + B * k2x + C * ux, ty = A * k1y + B * k2y + C * uy, tz = A * k1z + B * k2z + C * uz;
    lsd::Sim3 r;
    double rt[3];
    lsd::quatRotate(uq, T.t, rt);
    r.t[0] = tx + scale * rt[0]; r.t[1] = ty + scale * rt[1]; r.t[2] = tz + scale * rt[2];
    const double sq[4] = { scale * uq[0], scale * uq[1], scale * uq[2], scale * uq[3] };
    lsd::quatMul(sq, T.q, r.q);
    return r;
}
// lsd::sim3PoseConstants with one reciprocal for the quaternion normalisation
__device__ __forceinline__ void sim3PoseConstantsFast(const lsd::Sim3& a, float rotMat[9], float transVec[3], float roll[4])
{
    const double n2 = a.q[0] * a.q[0] + a.q[1] * a.q[1] + a.q[2] * a.q[2] + a.q[3] * a.q[3];
    const double scale = sqrt(n2), inv = 1.0 / scale;
    const double nq[4] = { a.q[0] * inv, a.q[1] * inv, a.q[2] * inv, a.q[3] * inv };
    double R[9];
    lsd::quatToMatrix(nq, R);
    float Ru[9];
#pragma unroll
    for (int i = 0; i < 9; i++) { rotMat[i] = (float)(scale * R[i]); Ru[i] = (float)R[i]; }
#pragma unroll
    for (int i = 0; i < 3; i++) transVec[i] = (float)a.t[i];
    // Sim3Tracker.cpp:451-460 (same steps as lsd::sim3PoseConstants)
    const float rf[3] = { -Ru[2], -Ru[5], -Ru[8] };
    const float n = sqrtf((rf[0] * rf[0] + rf[1] * rf[1]) + rf[2] * rf[2]);
    const float v0[3] = { rf[0] / n, rf[1] / n, rf[2] / n };
    const float c = -v0[2];
    if (c < -1.0f + 1e-5f) { roll[0] = roll[1] = roll[2] = roll[3] = nanf(""); return; }
    const float ax[3] = { v0[1] * -1.f - v0[2] * 0.f, v0[2] * 0.f - v0[0] * -1.f, v0[0] * 0.f - v0[1] * 0.f };
    const float s = sqrtf((1.f + c) * 2.f), invs = 1.f / s;
    const float q[4] = { ax[0] * invs, ax[1] * invs, ax[2] * invs, s * 0.5f };
    float Rb[9];
    lsd::quatToMatrix(q, Rb);
    roll[0] = (Rb[0] * Ru[0] + Rb[1] * Ru[3]) + Rb[2] * Ru[6];
    roll[1] = (Rb[0] * Ru[1] + Rb[1] * Ru[4]) + Rb[2] * Ru[7];
    roll[2] = (Rb[3] * Ru[0] + Rb[4] * Ru[3]) + Rb[5] * Ru[6];
    roll[3] = (Rb[3] * Ru[1] + Rb[4] * Ru[4]) + Rb[5] * Ru[7];
}

__device__ __forceinline__ void sim3SetPose(Sim3Shared& sh, const lsd::Sim3& T, float a, float b, int lvl)
{
    sim3PoseConstantsFast(T, sh.pose.R, sh.pose.t, sh.pose.roll);
    sh.pose.a = a; sh.pose.b = b;
    sh.lvl = lvl;
}

__device__ __noinline__ void sim3Advance(const Sim3Params& p, Sim3LM& lm, Sim3Shared& sh, const float* sums)
{
    const Sim3Res res = sim3Finish(sums);
    lm.pointUsage = res.pointUsage;
    const int lvl = lm.lvl;
    auto tooFew = [&](int l) { return res.warpedSize < 0.5 * 0.01f * (p.W >> l) * (p.H >> l) || res.warpedSize < 10; };   // :182, :229
    auto takeLGS = [&]() {
        for (int i = 0; i < S3_NLGS; i++) lm.lgs[i] = sums[i];
        lm.ncons = (float)(2 * res.warpedSize);
    };
    bool startIteration = false, propose = false, nextLevel = false;

    if (lm.phase == S3_PH_EVALONLY) { lm.done = 1; sh.done = 1; return; }
    if (lm.phase == S3_PH_FINAL) {                                                         // :351-358
        lm.resMean = res.mean; lm.resMeanD = res.meanD; lm.resMeanP = res.meanP;
        takeLGS();
        lm.done = 1; sh.done = 1;
        return;
    }
    if (lm.phase == S3_PH_INIT) {                                                          // :179-199
        if (tooFew(lvl)) { lm.early = 1; lm.done = 1; sh.done = 1; return; }
        lm.lastErrMean = res.mean;
        lm.nRes[lvl]++;
        if (p.useAffine) { lm.affine_a = res.a_lastIt; lm.affine_b = res.b_lastIt; }
        lm.LM_lambda = p.st.lambdaInitial[lvl];
        lm.warpUpToDate = 0;
        lm.iteration = 0;
        takeLGS();
        startIteration = true;
    } else {                                                                               // S3_PH_TRY, :226-311
        if (tooFew(lvl)) { lm.early = 1; lm.done = 1; sh.done = 1; return; }
        lm.nRes[lvl]++;
        if (res.mean < lm.lastErrMean) {
            lm.refToFrame = lm.cand;
            lm.warpUpToDate = 0;
            if (p.useAffine) { lm.affine_a = res.a_lastIt; lm.affine_b = res.b_lastIt; }
            if (res.mean / lm.lastErrMean > p.st.convergenceEps[lvl]) lm.iteration = p.st.maxItsPerLvl[lvl];
            lm.resMean = res.mean; lm.resMeanD = res.meanD; lm.resMeanP = res.meanP;
            lm.lastErrMean = res.mean;
            takeLGS();
            if (lm.LM_lambda <= 0.2) lm.LM_lambda = 0;
            else lm.LM_lambda *= p.st.lambdaSuccessFac;
            lm.iteration++;
            startIteration = true;
        } else {
            if (!(lm.absInc > p.st.stepSizeMin[lvl])) {
                lm.iteration = p.st.maxItsPerLvl[lvl] + 1;
                startIteration = true;
            } else {
                if (lm.LM_lambda == 0) lm.LM_lambda = 0.2;
                else lm.LM_lambda *= pow((double)p.st.lambdaFailFac, (double)lm.incTry);
                propose = true;
            }
        }
    }
    if (startIteration) {
        if (lm.iteration < p.st.maxItsPerLvl[lvl]) {                                       // :202-209
            lm.warpUpToDate = 1;
            lm.nUpd[lvl]++;
            lm.incTry = 0;
            propose = true;
        } else
            nextLevel = true;
    }
    if (propose) {                                                                         // :213-223
        float A7[49], b7[7], b[7], inc[7];
        sim3AssembleLGS7(lm.lgs, A7, b7);
        for (int i = 0; i < 7; i++) b[i] = -b7[i] / lm.ncons;
        for (int i = 0; i < 49; i++) A7[i] = A7[i] / lm.ncons;
        for (int i = 0; i < 7; i++) A7[i * 7 + i] *= 1 + lm.LM_lambda;
        if (!ldltSolveFast<7>(A7, b, inc)) lsd::ldltSolve<7>(A7, b, inc);
        lm.incTry++;
        float absInc = 0;
        for (int i = 0; i < 7; i++) absInc += inc[i] * inc[i];
        lm.absInc = absInc;
        if (!(absInc >= 0 && absInc < 1)) { lm.early = 2; lm.done = 1; sh.done = 1; return; }
        lm.cand = sim3ExpMulFast(inc, lm.refToFrame);
        lm.phase = S3_PH_TRY;
        sim3SetPose(sh, lm.cand, lm.affine_a, lm.affine_b, lvl);
        return;
    }
    if (nextLevel) {
        int l = lvl - 1;
        while (l >= p.finalLevel && p.st.maxItsPerLvl[l] == 0) l--;                        // :171-172
        if (l >= p.finalLevel) {
            lm.lvl = l; lm.phase = S3_PH_INIT;
            sim3SetPose(sh, lm.refToFrame, lm.affine_a, lm.affine_b, l);
        } else if (!lm.warpUpToDate) {
            lm.lvl = p.finalLevel; lm.phase = S3_PH_FINAL;
            sim3SetPose(sh, lm.refToFrame, lm.affine_a, lm.affine_b, p.finalLevel);
        } else {
            lm.done = 1; sh.done = 1;
        }
    }
}

// grid = nProblems * clusterSize CTAs, launched as clusters of clusterSize along x
__global__ void __launch_bounds__(S3_THREADS) k_sim3_track(const __grid_constant__ Sim3Params p, const Sim3Item* __restrict__ items,
                                                           Sim3Out* __restrict__ outs)
{
    cg::cluster_group cluster = cg::this_cluster();
    const int csize = (int)cluster.num_blocks(), crank = (int)cluster.block_rank();
    const int prob = blockIdx.x / csize;
    __shared__ alignas(Sim3LM) unsigned char lmStorage[sizeof(Sim3LM)];     // every field is written before use; no constructor in shared memory
    Sim3LM& lm = *reinterpret_cast<Sim3LM*>(lmStorage);
    __shared__ Sim3Shared sh;
    __shared__ float warpRows[S3_THREADS / 32][S3_NCH];
    __shared__ float xrow[2][S3_NCH];          // this CTA's partial sums, double-buffered by evaluation parity
    __shared__ float sums[S3_NCH];
    __shared__ int queue[S3_THREADS / 32][64];   // per-warp compaction queue of valid reference pixels
    const Sim3Item& it = items[prob];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    if (threadIdx.x == 0) {
        for (int i = 0; i < 4; i++) lm.refToFrame.q[i] = it.refToFrame[i];
        for (int i = 0; i < 3; i++) lm.refToFrame.t[i] = it.refToFrame[4 + i];
        for (int l = 0; l < LSD_LEVELS; l++) { lm.nRes[l] = 0; lm.nUpd[l] = 0; }
        for (int i = 0; i < S3_NLGS; i++) lm.lgs[i] = 0.f;
        lm.ncons = 1.f; lm.lastErrMean = 0.f; lm.resMean = lm.resMeanD = lm.resMeanP = 0.f;
        lm.affine_a = 1.f; lm.affine_b = 0.f; lm.LM_lambda = 0.f; lm.absInc = 0.f; lm.pointUsage = 0.f;
        lm.iteration = 0; lm.incTry = 0; lm.warpUpToDate = 0; lm.early = 0; lm.done = 0;
        sh.done = 0;
        if (p.evalOnly) {
            lm.lvl = p.startLevel; lm.phase = S3_PH_EVALONLY;
            lm.affine_a = p.evalA; lm.affine_b = p.evalB;
            sim3SetPose(sh, lm.refToFrame, lm.affine_a, lm.affine_b, lm.lvl);
        } else {
            int l = p.startLevel;
            while (l >= p.finalLevel && p.st.maxItsPerLvl[l] == 0) l--;
            if (l >= p.finalLevel) { lm.lvl = l; lm.phase = S3_PH_INIT; }
            else { lm.lvl = p.finalLevel; lm.phase = S3_PH_FINAL; }           // every level skipped: only the final warp update
            sim3SetPose(sh, lm.refToFrame, lm.affine_a, lm.affine_b, lm.lvl);
        }
    }
    __syncthreads();

    int parity = 0;
    long long cyc0 = 0, cyc1 = 0, cyc2 = 0, cyc3 = 0;
    while (true) {
        const long long tA = clock64();
        const int lvl = sh.lvl;
        const Sim3Pose P = sh.pose;
        const Sim3Level L = p.lvl[lvl];
        const float* __restrict__ kfIdepth = it.kfIdepth[lvl];
        const float* __restrict__ kfVar = it.kfVar[lvl];
        const float4* __restrict__ kfGrad = it.kfGrad[lvl];
        const float4* __restrict__ frGrad = it.frGrad[lvl];
        const float* __restrict__ frIdepth = it.frIdepth[lvl];
        const float* __restrict__ frVar = it.frVar[lvl];
        float acc[S3_NCH];
#pragma unroll
        for (int c = 0; c < S3_NCH; c++) acc[c] = 0.f;
        const int n = L.w * L.h;
        // Only ~40 % of the reference pixels carry a hypothesis (semi-dense map) and the per-point body is ~600 instructions:
        // each warp first compacts the indices of its valid pixels into a small shared-memory queue and runs the body on
        // full warps (same per-CTA compaction idea as k_observe).  The order is fixed by the data => still deterministic.
        auto body = [&](int i) {
            const int x = i % L.w, y = i / L.w;
            const float idepth = __ldg(kfIdepth + i), var = __ldg(kfVar + i);
            const float4 g = __ldg(kfGrad + i);
            const float sc = 1.0f / idepth;                                                // TrackingReference.cpp:135-136
            sim3EvalPoint(sc * (L.fxi * x + L.cxi), sc * (L.fyi * y + L.cyi), sc * 1, g.x, g.y, g.z, var, P, L, frGrad, frIdepth, frVar,
                          p.st.var_weight, p.st.huber_d, p.cameraPixelNoise2, acc);
        };
        int* q = queue[warp];
        int qCount = 0;
        for (int base = crank * S3_THREADS + warp * 32; base < n; base += csize * S3_THREADS) {      // warp-uniform trip count
            const int i = base + lane;
            bool valid = false;
            if (i < n) {
                const int x = i % L.w, y = i / L.w;
                if (!(x < 1 || x >= L.w - 1 || y < 1 || y >= L.h - 1)) {                   // TrackingReference.cpp:128-129
                    const float idepth = __ldg(kfIdepth + i), var = __ldg(kfVar + i);
                    valid = !(var <= 0 || idepth == 0);                                    // :133
                }
            }
            const unsigned int m = __ballot_sync(0xffffffffu, valid);
            if (valid) q[qCount + __popc(m & ((1u << lane) - 1u))] = i;
            qCount += __popc(m);
            __syncwarp();
            if (qCount >= 32) {
                body(q[lane]);
                __syncwarp();
                const int rest = qCount - 32;
                const int moved = lane < rest ? q[32 + lane] : 0;
                __syncwarp();
                if (lane < rest) q[lane] = moved;
                qCount = rest;
                __syncwarp();
            }
        }
        if (lane < qCount) body(q[lane]);
        const long long tB = clock64();
        // CTA reduction: 52 = 32 + 16 + 4 channels through the multi-value butterfly (53 shuffles instead of 260), then one
        // shared-memory stage in fixed order
        {
            float a32[32], a16[16], a4[4];
#pragma unroll
            for (int i = 0; i < 32; i++) a32[i] = acc[i];
#pragma unroll
            for (int i = 0; i < 16; i++) a16[i] = acc[32 + i];
#pragma unroll
            for (int i = 0; i < 4; i++) a4[i] = acc[48 + i];
            warpReduceMulti<32>(a32, lane);
            warpReduceMulti<16>(a16, lane);
            warpReduceMulti<4>(a4, lane);
            warpRows[warp][lane] = a32[0];
            if ((lane & 1) == 0) warpRows[warp][32 + warpReduceChannel<16>(lane)] = a16[0];
            if ((lane & 7) == 0) warpRows[warp][48 + warpReduceChannel<4>(lane)] = a4[0];
        }
        __syncthreads();
        if (threadIdx.x < S3_NCH) {
            float s = 0.f;
#pragma unroll
            for (int wi = 0; wi < S3_THREADS / 32; wi++) s += warpRows[wi][threadIdx.x];
            xrow[parity][threadIdx.x] = s;
        }
        const long long tC = clock64();
        // cluster exchange: every CTA sums the rows of all ranks in rank order -> identical totals everywhere
        if (csize > 1) cluster.sync(); else __syncthreads();
        if (threadIdx.x < S3_NCH) {
            float tot = 0.f;
            for (int r = 0; r < csize; r++) tot += cluster.map_shared_rank(&xrow[parity][0], r)[threadIdx.x];
            sums[threadIdx.x] = tot;
        }
        __syncthreads();
        const long long tD = clock64();
        if (threadIdx.x == 0) sim3Advance(p, lm, sh, sums);
        __syncthreads();
        const long long tE = clock64();
        cyc0 += tB - tA; cyc1 += tC - tB; cyc2 += tD - tC; cyc3 += tE - tD;
        parity ^= 1;
        if (sh.done) break;
    }
    if (csize > 1) cluster.sync();              // nobody may exit while a peer can still read its xrow
    if (crank == 0 && threadIdx.x < S3_NCH) outs[prob].sums[threadIdx.x] = sums[threadIdx.x];
    if (crank == 0 && threadIdx.x == 0) {
        Sim3Out& o = outs[prob];
        for (int i = 0; i < 4; i++) o.refToFrame[i] = lm.refToFrame.q[i];
        for (int i = 0; i < 3; i++) o.refToFrame[4 + i] = lm.refToFrame.t[i];
        for (int i = 0; i < S3_NLGS; i++) o.lgs[i] = lm.lgs[i];
        o.resMean = lm.resMean; o.resMeanD = lm.resMeanD; o.resMeanP = lm.resMeanP;
        o.pointUsage = lm.pointUsage; o.affine_a = lm.affine_a; o.affine_b = lm.affine_b;
        o.early = lm.early;
        for (int l = 0; l < LSD_LEVELS; l++) { o.nRes[l] = lm.nRes[l]; o.nUpd[l] = lm.nUpd[l]; }
        o.cyc[0] = cyc0; o.cyc[1] = cyc1; o.cyc[2] = cyc2; o.cyc[3] = cyc3;
    }
}
