// depth.cuh -- per-pixel kernels of DepthMap (semi-dense inverse-depth filter).
//
// Replaces (paths relative to lsd_slam_core/src/DepthEstimation/DepthMap.cpp):
//   observeDepthRow / Create / Update      :111-146, 237-292, 294-473      -> k_observe
//   makeAndCheckEPL                        :184-234
//   doLineStereo                           :1442-1972   (NDEBUG semantics: enablePrintDebugInfo == false)
//   buildRegIntegralBuffer + FillHolesRow  :722-754, 656-703               -> k_fill_holes (5x5 validity sum
//                                          taken directly; the integral image is never needed on the GPU)
//   regularizeDepthMapRow<removeOcclusions>:758-848                        -> k_regularize<bool>
//   propagateDepth                         :475-653                        -> k_prop_project + k_prop_resolve
//   createKeyFrame rescale                 :1285-1304                      -> seqsum.cuh (the sequential fp32 sum) + k_rescale
//   Frame::setDepth                        DataStructures/Frame.cpp:199-243 -> k_set_depth_pyr, or the SETDEPTH stage
//                                                                              of k_fill_regularize
//   Frame::takeReActivationData            DataStructures/Frame.cpp:107-145 -> k_take_reactivation
//   setFromExistingKF                      :920-962                        -> k_set_from_existing
// The reference's memcpy(other <- current) + read other / write current (:713, :862) is a ping-pong here:
// every kernel reads `src` and writes every pixel of `dst`.
//
// Arithmetic is kept in the reference's order and the library is compiled with --fmad=false, so per-pixel
// results are bit-identical to a strict-IEEE CPU evaluation (threshold decisions included).
#pragma once
#include "internal.cuh"

#define DIVISION_EPS 1e-10f
#define VALIDITY_COUNTER_MAX (5.0f)
#define VALIDITY_COUNTER_MAX_VARIABLE (250.0f)
#define VALIDITY_COUNTER_INC 5
#define VALIDITY_COUNTER_DEC 5
#define VALIDITY_COUNTER_INITIAL_OBSERVE 5
#define VAL_SUM_MIN_FOR_CREATE (30)
#define VAL_SUM_MIN_FOR_KEEP (24)
#define VAL_SUM_MIN_FOR_UNBLACKLIST (100)
#define MIN_BLACKLIST -1
#define SUCC_VAR_INC_FAC (1.01f)
#define FAIL_VAR_INC_FAC 1.1f
#define MAX_VAR (0.5f*0.5f)
#define VAR_RANDOM_INIT_INITIAL (0.5f*MAX_VAR)
#define MIN_DEPTH 0.05f
#define MAX_EPL_LENGTH_CROP 30.0f
#define MIN_EPL_LENGTH_CROP (3.0f)
#define GRADIENT_SAMPLE_DIST 1.0f
#define SAMPLE_POINT_TO_BORDER 7
#define MAX_ERROR_STEREO (1300.0f)
#define MIN_DISTANCE_ERROR_STEREO (1.5f)
#define STEREO_EPL_VAR_FAC 2.0f
#define DIFF_FAC_SMOOTHING (1.0f*1.0f)
#define DIFF_FAC_OBSERVE (1.0f*1.0f)
#define DIFF_FAC_PROP_MERGE (1.0f*1.0f)
#define MIN_EPL_GRAD_SQUARED (2.0f*2.0f)
#define MIN_EPL_LENGTH_SQUARED (1.0f*1.0f)
#define MIN_EPL_ANGLE_SQUARED (0.3f*0.3f)
#define MAX_DIFF_CONSTANT (40.0f*40.0f)
#define MAX_DIFF_GRAD_MULT (0.5f*0.5f)

struct DepthCam {
    int w, h;
    float fx, fy, cx, cy, fxi, fyi, cxi, cyi;
};
struct DepthGlobals {
    float minUseGrad, cameraPixelNoise2, regDistVar;
    int allowNegativeIdepths, useSubpixelStereo;
};

// hypothesis record in registers; hf/hi planes, see internal.cuh
struct Hyp {
    int isValid, blacklisted, validity_counter;
    float nextStereoFrameMinID;
    float idepth, idepth_var, idepth_smoothed, idepth_var_smoothed;
};
__device__ __forceinline__ Hyp loadHyp(const HypField& f, int i)
{
    float4 a = f.hf[i];
    int4 b = f.hi[i];
    Hyp h;
    h.idepth = a.x; h.idepth_var = a.y; h.idepth_smoothed = a.z; h.idepth_var_smoothed = a.w;
    h.isValid = b.x; h.blacklisted = b.y; h.validity_counter = b.z; h.nextStereoFrameMinID = __int_as_float(b.w);
    return h;
}
__device__ __forceinline__ void storeHyp(const HypField& f, int i, const Hyp& h)
{
    f.hf[i] = make_float4(h.idepth, h.idepth_var, h.idepth_smoothed, h.idepth_var_smoothed);
    f.hi[i] = make_int4(h.isValid, h.blacklisted, h.validity_counter, __float_as_int(h.nextStereoFrameMinID));
}
// DepthMapPixelHypothesis(idepth, var, validity), DepthMapPixelHypothesis.h:80-91
__device__ __forceinline__ void hypCtor3(Hyp& h, float idepth, float var, int validity)
{
    h.isValid = 1; h.blacklisted = 0; h.nextStereoFrameMinID = 0; h.validity_counter = validity;
    h.idepth = idepth; h.idepth_var = var; h.idepth_smoothed = -1; h.idepth_var_smoothed = -1;
}

// ---------------------------------------------------------------------------------------------------------
// doLineStereo, DepthMap.cpp:1442-1972.  Returns the reference's error code / SSD.
// ---------------------------------------------------------------------------------------------------------
__device__ __noinline__ float doLineStereo(
    const DepthCam& cam, const DepthGlobals& G, const float* __restrict__ kfImage, const float4* __restrict__ kfGrad,
    const float u, const float v, const float epxn, const float epyn,
    const float min_idepth, const float prior_idepth, float max_idepth,
    const RefConst& ref, float& result_idepth, float& result_var, float& result_eplLength)
{
    const int width = cam.w, height = cam.h;
    const float fxi = cam.fxi, fyi = cam.fyi, cxi = cam.cxi, cyi = cam.cyi;
    const float* __restrict__ refImage = ref.image;
    const float* KR = ref.K_otherToThis_R;
    const float* Kt = ref.K_otherToThis_t;

    float KinvP[3] = { fxi * u + cxi, fyi * v + cyi, 1.0f };
    float pInf[3], pReal[3];
#pragma unroll
    for (int i = 0; i < 3; i++) pInf[i] = (KR[i * 3 + 0] * KinvP[0] + KR[i * 3 + 1] * KinvP[1]) + KR[i * 3 + 2] * KinvP[2];
#pragma unroll
    for (int i = 0; i < 3; i++) pReal[i] = pInf[i] / prior_idepth + Kt[i];

    float rescaleFactor = pReal[2] * prior_idepth;

    float firstX = u - 2 * epxn * rescaleFactor;
    float firstY = v - 2 * epyn * rescaleFactor;
    float lastX = u + 2 * epxn * rescaleFactor;
    float lastY = v + 2 * epyn * rescaleFactor;
    if (firstX <= 0 || firstX >= width - 2 || firstY <= 0 || firstY >= height - 2
        || lastX <= 0 || lastX >= width - 2 || lastY <= 0 || lastY >= height - 2)
        return -1;
    if (!(rescaleFactor > 0.7f && rescaleFactor < 1.4f)) return -1;

    float realVal_p1 = interpF(kfImage, u + epxn * rescaleFactor, v + epyn * rescaleFactor, width);
    float realVal_m1 = interpF(kfImage, u - epxn * rescaleFactor, v - epyn * rescaleFactor, width);
    float realVal = interpF(kfImage, u, v, width);
    float realVal_m2 = interpF(kfImage, u - 2 * epxn * rescaleFactor, v - 2 * epyn * rescaleFactor, width);
    float realVal_p2 = interpF(kfImage, u + 2 * epxn * rescaleFactor, v + 2 * epyn * rescaleFactor, width);

    float pClose[3], pFar[3];
#pragma unroll
    for (int i = 0; i < 3; i++) pClose[i] = pInf[i] + Kt[i] * max_idepth;
    if (pClose[2] < 0.001f) {
        max_idepth = (0.001f - pInf[2]) / Kt[2];
#pragma unroll
        for (int i = 0; i < 3; i++) pClose[i] = pInf[i] + Kt[i] * max_idepth;
    }
    { float z = pClose[2]; pClose[0] = pClose[0] / z; pClose[1] = pClose[1] / z; pClose[2] = pClose[2] / z; }

#pragma unroll
    for (int i = 0; i < 3; i++) pFar[i] = pInf[i] + Kt[i] * min_idepth;
    if (pFar[2] < 0.001f || max_idepth < min_idepth) return -1;
    { float z = pFar[2]; pFar[0] = pFar[0] / z; pFar[1] = pFar[1] / z; pFar[2] = pFar[2] / z; }

    if (isnan((float)(pFar[0] + pClose[0]))) return -4;

    float incx = pClose[0] - pFar[0];
    float incy = pClose[1] - pFar[1];
    float eplLength = sqrtf(incx * incx + incy * incy);
    if ((eplLength == 0.0f) || isinf(eplLength)) return -4;       // `!eplLength > 0` parses as (!eplLength) > 0, :1518

    if (eplLength > MAX_EPL_LENGTH_CROP) {
        pClose[0] = pFar[0] + incx * MAX_EPL_LENGTH_CROP / eplLength;
        pClose[1] = pFar[1] + incy * MAX_EPL_LENGTH_CROP / eplLength;
    }

    incx *= GRADIENT_SAMPLE_DIST / eplLength;
    incy *= GRADIENT_SAMPLE_DIST / eplLength;

    pFar[0] -= incx; pFar[1] -= incy;
    pClose[0] += incx; pClose[1] += incy;

    if (eplLength < MIN_EPL_LENGTH_CROP) {
        float pad = (MIN_EPL_LENGTH_CROP - (eplLength)) / 2.0f;
        pFar[0] -= incx * pad; pFar[1] -= incy * pad;
        pClose[0] += incx * pad; pClose[1] += incy * pad;
    }

    if (pFar[0] <= SAMPLE_POINT_TO_BORDER || pFar[0] >= width - SAMPLE_POINT_TO_BORDER ||
        pFar[1] <= SAMPLE_POINT_TO_BORDER || pFar[1] >= height - SAMPLE_POINT_TO_BORDER)
        return -1;

    if (pClose[0] <= SAMPLE_POINT_TO_BORDER || pClose[0] >= width - SAMPLE_POINT_TO_BORDER ||
        pClose[1] <= SAMPLE_POINT_TO_BORDER || pClose[1] >= height - SAMPLE_POINT_TO_BORDER) {
        if (pClose[0] <= SAMPLE_POINT_TO_BORDER) {
            float toAdd = (SAMPLE_POINT_TO_BORDER - pClose[0]) / incx;
            pClose[0] += toAdd * incx; pClose[1] += toAdd * incy;
        } else if (pClose[0] >= width - SAMPLE_POINT_TO_BORDER) {
            float toAdd = (width - SAMPLE_POINT_TO_BORDER - pClose[0]) / incx;
            pClose[0] += toAdd * incx; pClose[1] += toAdd * incy;
        }
        if (pClose[1] <= SAMPLE_POINT_TO_BORDER) {
            float toAdd = (SAMPLE_POINT_TO_BORDER - pClose[1]) / incy;
            pClose[0] += toAdd * incx; pClose[1] += toAdd * incy;
        } else if (pClose[1] >= height - SAMPLE_POINT_TO_BORDER) {
            float toAdd = (height - SAMPLE_POINT_TO_BORDER - pClose[1]) / incy;
            pClose[0] += toAdd * incx; pClose[1] += toAdd * incy;
        }
        float fincx = pClose[0] - pFar[0];
        float fincy = pClose[1] - pFar[1];
        float newEplLength = sqrtf(fincx * fincx + fincy * fincy);
        if (pClose[0] <= SAMPLE_POINT_TO_BORDER || pClose[0] >= width - SAMPLE_POINT_TO_BORDER ||
            pClose[1] <= SAMPLE_POINT_TO_BORDER || pClose[1] >= height - SAMPLE_POINT_TO_BORDER ||
            newEplLength < 8.0f)
            return -1;
    }

    float cpx = pFar[0];
    float cpy = pFar[1];

    float val_cp_m2 = interpF(refImage, cpx - 2.0f * incx, cpy - 2.0f * incy, width);
    float val_cp_m1 = interpF(refImage, cpx - incx, cpy - incy, width);
    float val_cp = interpF(refImage, cpx, cpy, width);
    float val_cp_p1 = interpF(refImage, cpx + incx, cpy + incy, width);
    float val_cp_p2;

    const float fNAN = __int_as_float(0x7fc00000);
    const float fINF = __int_as_float(0x7f800000);
    int loopCounter = 0;
    float best_match_x = -1;
    float best_match_y = -1;
    float best_match_err = fINF;                 // `float x = 1e50` -> +inf, :1658-1659
    float second_best_match_err = fINF;
    float best_match_errPre = fNAN, best_match_errPost = fNAN, best_match_DiffErrPre = fNAN, best_match_DiffErrPost = fNAN;
    bool bestWasLastLoop = false;
    float eeLast = -1;
    float e1A = fNAN, e1B = fNAN, e2A = fNAN, e2B = fNAN, e3A = fNAN, e3B = fNAN, e4A = fNAN, e4B = fNAN, e5A = fNAN, e5B = fNAN;
    int loopCBest = -1, loopCSecond = -1;

    // the reference loop has no bound; with finite inputs it ends after <= ~40 steps (30-px crop + padding).
    // 4096 only protects the GPU from a NaN-poisoned frame (where the reference would spin forever).
    while ((((incx < 0) == (cpx > pClose[0]) && (incy < 0) == (cpy > pClose[1])) || loopCounter == 0) && loopCounter < 4096) {
        val_cp_p2 = interpF(refImage, cpx + 2 * incx, cpy + 2 * incy, width);
        float ee = 0;
        if (loopCounter % 2 == 0) {
            e1A = val_cp_p2 - realVal_p2; ee += e1A * e1A;
            e2A = val_cp_p1 - realVal_p1; ee += e2A * e2A;
            e3A = val_cp - realVal;       ee += e3A * e3A;
            e4A = val_cp_m1 - realVal_m1; ee += e4A * e4A;
            e5A = val_cp_m2 - realVal_m2; ee += e5A * e5A;
        } else {
            e1B = val_cp_p2 - realVal_p2; ee += e1B * e1B;
            e2B = val_cp_p1 - realVal_p1; ee += e2B * e2B;
            e3B = val_cp - realVal;       ee += e3B * e3B;
            e4B = val_cp_m1 - realVal_m1; ee += e4B * e4B;
            e5B = val_cp_m2 - realVal_m2; ee += e5B * e5B;
        }
        if (ee < best_match_err) {
            second_best_match_err = best_match_err;
            loopCSecond = loopCBest;
            best_match_err = ee;
            loopCBest = loopCounter;
            best_match_errPre = eeLast;
            best_match_DiffErrPre = e1A * e1B + e2A * e2B + e3A * e3B + e4A * e4B + e5A * e5B;
            best_match_errPost = -1;
            best_match_DiffErrPost = -1;
            best_match_x = cpx;
            best_match_y = cpy;
            bestWasLastLoop = true;
        } else {
            if (bestWasLastLoop) {
                best_match_errPost = ee;
                best_match_DiffErrPost = e1A * e1B + e2A * e2B + e3A * e3B + e4A * e4B + e5A * e5B;
                bestWasLastLoop = false;
            }
            if (ee < second_best_match_err) {
                second_best_match_err = ee;
                loopCSecond = loopCounter;
            }
        }
        eeLast = ee;
        val_cp_m2 = val_cp_m1; val_cp_m1 = val_cp; val_cp = val_cp_p1; val_cp_p1 = val_cp_p2;
        cpx += incx;
        cpy += incy;
        loopCounter++;
    }

    if (best_match_err > 4.0f * (float)MAX_ERROR_STEREO) return -3;

    if (abs(loopCBest - loopCSecond) > 1.0f && MIN_DISTANCE_ERROR_STEREO * best_match_err > second_best_match_err) return -2;

    bool didSubpixel = false;
    if (G.useSubpixelStereo) {
        float gradPre_pre = -(best_match_errPre - best_match_DiffErrPre);
        float gradPre_this = +(best_match_err - best_match_DiffErrPre);
        float gradPost_this = -(best_match_err - best_match_DiffErrPost);
        float gradPost_post = +(best_match_errPost - best_match_DiffErrPost);
        bool interpPost = false, interpPre = false;
        if ((gradPost_this < 0) ^ (gradPre_this < 0)) {
        } else if ((gradPre_pre < 0) ^ (gradPre_this < 0)) {
            if ((gradPost_post < 0) ^ (gradPost_this < 0)) {
            } else
                interpPre = true;
        } else if ((gradPost_post < 0) ^ (gradPost_this < 0)) {
            interpPost = true;
        }
        if (interpPre) {
            float d = gradPre_this / (gradPre_this - gradPre_pre);
            best_match_x -= d * incx;
            best_match_y -= d * incy;
            best_match_err = best_match_err - 2 * d * gradPre_this - (gradPre_pre - gradPre_this) * d * d;
            didSubpixel = true;
        } else if (interpPost) {
            float d = gradPost_this / (gradPost_this - gradPost_post);
            best_match_x += d * incx;
            best_match_y += d * incy;
            best_match_err = best_match_err + 2 * d * gradPost_this + (gradPost_post - gradPost_this) * d * d;
            didSubpixel = true;
        }
    }

    float sampleDist = GRADIENT_SAMPLE_DIST * rescaleFactor;

    float gradAlongLine = 0;
    float tmp = realVal_p2 - realVal_p1; gradAlongLine += tmp * tmp;
    tmp = realVal_p1 - realVal; gradAlongLine += tmp * tmp;
    tmp = realVal - realVal_m1; gradAlongLine += tmp * tmp;
    tmp = realVal_m1 - realVal_m2; gradAlongLine += tmp * tmp;
    gradAlongLine /= sampleDist * sampleDist;

    if (best_match_err > (float)MAX_ERROR_STEREO + sqrtf(gradAlongLine) * 20) return -3;

    float idnew_best_match, alpha;
    const float* oTt = ref.otherToThis_t;
#define DOT3(a, b) ((a)[0] * (b)[0] + ((a)[1] * (b)[1] + (a)[2] * (b)[2]))
    if (incx * incx > incy * incy) {
        float oldX = fxi * best_match_x + cxi;
        float nominator = (oldX * oTt[2] - oTt[0]);
        float dot0 = DOT3(KinvP, ref.row0);
        float dot2 = DOT3(KinvP, ref.row2);
        idnew_best_match = (dot0 - oldX * dot2) / nominator;
        alpha = incx * fxi * (dot0 * oTt[2] - dot2 * oTt[0]) / (nominator * nominator);
    } else {
        float oldY = fyi * best_match_y + cyi;
        float nominator = (oldY * oTt[2] - oTt[1]);
        float dot1 = DOT3(KinvP, ref.row1);
        float dot2 = DOT3(KinvP, ref.row2);
        idnew_best_match = (dot1 - oldY * dot2) / nominator;
        alpha = incy * fyi * (dot1 * oTt[2] - dot2 * oTt[1]) / (nominator * nominator);
    }
#undef DOT3

    if (idnew_best_match < 0) {
        if (!G.allowNegativeIdepths) return -2;
    }

    float photoDispError = 4.0f * G.cameraPixelNoise2 / (gradAlongLine + DIVISION_EPS);
    float trackingErrorFac = 0.25f * (1.0f + ref.initialTrackedResidual);

    // getInterpolatedElement42(gradients(0), u, v): u, v are integer pixel coordinates here, the bilinear
    // weights are (0,0,0,1); evaluated in the reference's order so that the value is bit-identical
    float gI0, gI1;
    {
        int ix = (int)u, iy = (int)v;
        float dx = u - ix, dy = v - iy;
        float dxdy = dx * dy;
        const float4* bp = kfGrad + ix + iy * width;
        float4 br = __ldg(bp + 1 + width), bl = __ldg(bp + width), tr = __ldg(bp + 1), tl = __ldg(bp);
        gI0 = dxdy * br.x + (dy - dxdy) * bl.x + (dx - dxdy) * tr.x + (1 - dx - dy + dxdy) * tl.x;
        gI1 = dxdy * br.y + (dy - dxdy) * bl.y + (dx - dxdy) * tr.y + (1 - dx - dy + dxdy) * tl.y;
    }
    float geoDispError = (gI0 * epxn + gI1 * epyn) + DIVISION_EPS;
    geoDispError = trackingErrorFac * trackingErrorFac * (gI0 * gI0 + gI1 * gI1) / (geoDispError * geoDispError);

    result_var = alpha * alpha * ((didSubpixel ? 0.05f : 0.5f) * sampleDist * sampleDist + geoDispError + photoDispError);
    result_idepth = idnew_best_match;
    result_eplLength = eplLength;
    return best_match_err;
}

// makeAndCheckEPL, DepthMap.cpp:184-234
__device__ __forceinline__ bool makeAndCheckEPL(const DepthCam& cam, const float* __restrict__ kfImage, int x, int y,
                                                const RefConst& ref, float& pepx, float& pepy)
{
    int idx = x + y * cam.w;
    float epx = -cam.fx * ref.thisToOther_t[0] + ref.thisToOther_t[2] * (x - cam.cx);
    float epy = -cam.fy * ref.thisToOther_t[1] + ref.thisToOther_t[2] * (y - cam.cy);
    if (isnan(epx + epy)) return false;
    float eplLengthSquared = epx * epx + epy * epy;
    if (eplLengthSquared < MIN_EPL_LENGTH_SQUARED) return false;
    float gx = kfImage[idx + 1] - kfImage[idx - 1];
    float gy = kfImage[idx + cam.w] - kfImage[idx - cam.w];
    float eplGradSquared = gx * epx + gy * epy;
    eplGradSquared = eplGradSquared * eplGradSquared / eplLengthSquared;
    if (eplGradSquared < MIN_EPL_GRAD_SQUARED) return false;
    if (eplGradSquared / (gx * gx + gy * gy) < MIN_EPL_ANGLE_SQUARED) return false;
    float fac = GRADIENT_SAMPLE_DIST / sqrtf(eplLengthSquared);
    pepx = epx * fac;
    pepy = epy * fac;
    return true;
}

// observeDepthRow + Create + Update, DepthMap.cpp:111-146, 237-292, 294-473.  In place on `cur`: every pixel touches
// only its own record.
//
// The work is sparse and very uneven (about 40 % of the pixels pass the gates, and the line search runs 5-40 steps), so a
// CTA first runs the cheap gates for its OBS_PIX_PER_CTA pixels (3 per thread, coalesced), collects the survivors in a shared-memory
// list, and then walks that list densely: warps stay full during the expensive doLineStereo part.  The per-pixel
// arithmetic is untouched (the list order does not matter: pixels are independent).
#define OBS_THREADS 768
#define OBS_PIX_PER_CTA 2304          // 3 per thread; 640x480: 131 CTAs = one wave of 1 CTA per SM on H100's 132 SMs

// gates of observeDepthRow (:124-132) and of observeDepthCreate / Update up to and including makeAndCheckEPL
// (:241-256, :300-333).  Returns the reference index (>= 0) if the pixel must run the line search, -1 otherwise.
__device__ __forceinline__ int observeGate(const HypField& cur, const DepthCam& cam, const DepthGlobals& G,
                                           const float* __restrict__ kfImage, const float* __restrict__ kfMaxGrad,
                                           const ObserveParams* __restrict__ OP, int x, int y, int idx, float& epx, float& epy)
{
    int4 hiv = cur.hi[idx];
    const bool hasHypothesis = hiv.x != 0;
    const float mg = kfMaxGrad[idx];
    if (hasHypothesis && mg < G.minUseGrad) {              // :125-129
        hiv.x = 0;
        cur.hi[idx] = hiv;
        return -1;
    }
    if (mg < G.minUseGrad || hiv.y < MIN_BLACKLIST) return -1;   // :131-132
    int refIdx;
    if (!hasHypothesis) {
        refIdx = OP->reactivated ? OP->newestIdx : OP->oldestIdx;                 // :241
    } else {
        if (!OP->reactivated) {                                                   // :300-317
            const int rel = (int)__int_as_float(hiv.w) - OP->byIdOffset;
            if (rel >= OP->byIdSize) return -1;
            refIdx = rel < 0 ? OP->oldestIdx : OP->byId[rel];
        } else
            refIdx = OP->newestIdx;
    }
    const RefConst& ref = OP->refs[refIdx];
    if (ref.trackedOnActive && ref.goodMask != nullptr &&
        !ref.goodMask[(x >> SE3TRACKING_MIN_LEVEL) + (cam.w >> SE3TRACKING_MIN_LEVEL) * (y >> SE3TRACKING_MIN_LEVEL)])
        return -1;                                                                 // :243-252 / :320-329
    if (!makeAndCheckEPL(cam, kfImage, x, y, ref, epx, epy)) return -1;
    return refIdx;
}

// line search + hypothesis create / EKF update for one surviving pixel (:254-291, :335-472)
__device__ __forceinline__ void observeStereo(const HypField& cur, const DepthCam& cam, const DepthGlobals& G,
                                              const float* __restrict__ kfImage, const float4* __restrict__ kfGrad,
                                              const float* __restrict__ kfMaxGrad, const ObserveParams* __restrict__ OP,
                                              int x, int y, int idx, int refIdx, float epx, float epy)
{
    const RefConst& ref = OP->refs[refIdx];
    Hyp t = loadHyp(cur, idx);
    const bool hasHypothesis = t.isValid != 0;
    float result_idepth = 0, result_var = 0, result_eplLength = 0;
    if (!hasHypothesis) {
        // observeDepthCreate :254-291
        float error = doLineStereo(cam, G, kfImage, kfGrad, (float)x, (float)y, epx, epy, 0.0f, 1.0f, 1.0f / MIN_DEPTH,
                                   ref, result_idepth, result_var, result_eplLength);
        if (error == -3 || error == -2) {
            int4 hiv = cur.hi[idx];
            hiv.y = t.blacklisted - 1;
            cur.hi[idx] = hiv;
        }
        if (error < 0 || result_var > MAX_VAR) return;
        result_idepth = unzero_f(result_idepth);
        hypCtor3(t, result_idepth, result_var, VALIDITY_COUNTER_INITIAL_OBSERVE);
        storeHyp(cur, idx, t);
        return;
    }

    // observeDepthUpdate :335-472
    float sv = sqrtf(t.idepth_var_smoothed);
    float min_idepth = t.idepth_smoothed - sv * STEREO_EPL_VAR_FAC;
    float max_idepth = t.idepth_smoothed + sv * STEREO_EPL_VAR_FAC;
    if (min_idepth < 0) min_idepth = 0;
    if (max_idepth > 1 / MIN_DEPTH) max_idepth = 1 / MIN_DEPTH;

    float error = doLineStereo(cam, G, kfImage, kfGrad, (float)x, (float)y, epx, epy, min_idepth, t.idepth_smoothed, max_idepth,
                               ref, result_idepth, result_var, result_eplLength);
    float diff = result_idepth - t.idepth_smoothed;

    if (error == -1) return;
    else if (error == -2) {
        t.validity_counter -= VALIDITY_COUNTER_DEC;
        if (t.validity_counter < 0) t.validity_counter = 0;
        t.nextStereoFrameMinID = 0;
        t.idepth_var *= FAIL_VAR_INC_FAC;
        if (t.idepth_var > MAX_VAR) { t.isValid = 0; t.blacklisted--; }
        storeHyp(cur, idx, t);
        return;
    } else if (error == -3) return;
    else if (error == -4) return;
    else if (DIFF_FAC_OBSERVE * diff * diff > result_var + t.idepth_var_smoothed) {
        t.idepth_var *= FAIL_VAR_INC_FAC;
        if (t.idepth_var > MAX_VAR) t.isValid = 0;
        storeHyp(cur, idx, t);
        return;
    } else {
        float id_var = t.idepth_var * SUCC_VAR_INC_FAC;
        float w = result_var / (result_var + id_var);
        float new_idepth = (1 - w) * result_idepth + w * t.idepth;
        t.idepth = unzero_f(new_idepth);
        id_var = id_var * w;
        if (id_var < t.idepth_var) t.idepth_var = id_var;
        t.validity_counter += VALIDITY_COUNTER_INC;
        float absGrad = kfMaxGrad[idx];
        if (t.validity_counter > VALIDITY_COUNTER_MAX + absGrad * (VALIDITY_COUNTER_MAX_VARIABLE) / 255.0f)
            t.validity_counter = VALIDITY_COUNTER_MAX + absGrad * (VALIDITY_COUNTER_MAX_VARIABLE) / 255.0f;
        if (result_eplLength < MIN_EPL_LENGTH_CROP) {
            float inc = OP->kfNumTracked / (float)(OP->kfNumMapped + 5);
            if (inc < 3) inc = 3;
            inc += ((int)(result_eplLength * 10000) % 2);
            if (result_eplLength < 0.5 * MIN_EPL_LENGTH_CROP) inc *= 3;
            t.nextStereoFrameMinID = ref.id + inc;
        }
        storeHyp(cur, idx, t);
    }
}

__global__ void __launch_bounds__(OBS_THREADS) k_observe(HypField cur, DepthCam cam, DepthGlobals G,
                                                 const float* __restrict__ kfImage, const float4* __restrict__ kfGrad,
                                                 const float* __restrict__ kfMaxGrad, const __grid_constant__ ObserveParams OPv)
{
    __shared__ int sList[OBS_PIX_PER_CTA];
    __shared__ int sCount;
    pdlWait();                                       // launched early (programmatic dependent launch): wait for the tracking kernel
    const ObserveParams* OP = &OPv;
    const int iw = cam.w - 6, ih = cam.h - 6;        // x in [3, w-3), y in [3, h-3)  (:118, :150)
    const int nInterior = iw * ih;
    if (threadIdx.x == 0) sCount = 0;
    __syncthreads();
    const int base = blockIdx.x * OBS_PIX_PER_CTA;
    for (int jj = threadIdx.x; jj < OBS_PIX_PER_CTA; jj += OBS_THREADS) {
        const int j = base + jj;
        if (j < nInterior) {
            const int x = 3 + j % iw, y = 3 + j / iw;
            const int idx = x + y * cam.w;
            float epx, epy;
            const int refIdx = observeGate(cur, cam, G, kfImage, kfMaxGrad, OP, x, y, idx, epx, epy);
            if (refIdx >= 0) sList[atomicAdd(&sCount, 1)] = idx;
        }
    }
    __syncthreads();
    const int n = sCount;
    for (int e = threadIdx.x; e < n; e += OBS_THREADS) {
        const int idx = sList[e];
        const int x = idx % cam.w, y = idx / cam.w;
        float epx, epy;
        // the gates are re-evaluated (cheap, same inputs: nothing this pixel reads has been written in between)
        const int refIdx = observeGate(cur, cam, G, kfImage, kfMaxGrad, OP, x, y, idx, epx, epy);
        if (refIdx >= 0) observeStereo(cur, cam, G, kfImage, kfGrad, kfMaxGrad, OP, x, y, idx, refIdx, epx, epy);
    }
}

// regularizeDepthMapFillHoles, DepthMap.cpp:656-718.  dst = src + created hypotheses.
__global__ void __launch_bounds__(256) k_fill_holes(HypField src, HypField dst, DepthCam cam, DepthGlobals G,
                                                    const float* __restrict__ kfMaxGrad)
{
    const int x = blockIdx.x * 32 + (threadIdx.x & 31);
    const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= cam.w || y >= cam.h) return;
    const int width = cam.w;
    const int idx = x + y * width;
    float4 hf = src.hf[idx];
    int4 hi = src.hi[idx];
    if (x >= 3 && x < width - 2 && y >= 3 && y < cam.h - 2 && !hi.x && !(kfMaxGrad[idx] < G.minUseGrad)) {
        // val = 5x5 sum of (isValid ? validity_counter : 0) == the integral-image lookup of :670-671
        int val = 0;
        for (int dy = -2; dy <= 2; dy++)
            for (int dx = -2; dx <= 2; dx++) {
                int4 s = src.hi[idx + dx + dy * width];
                if (s.x) val += s.z;
            }
        if ((hi.y >= MIN_BLACKLIST && val > VAL_SUM_MIN_FOR_CREATE) || val > VAL_SUM_MIN_FOR_UNBLACKLIST) {
            float sumIdepthObs = 0, sumIVarObs = 0;
            for (int dy = -2; dy <= 2; dy++)             // row-major source order, :679-688
                for (int dx = -2; dx <= 2; dx++) {
                    int o = idx + dx + dy * width;
                    if (!src.hi[o].x) continue;
                    float4 s = src.hf[o];
                    sumIdepthObs += s.x / s.y;
                    sumIVarObs += 1.0f / s.y;
                }
            float idepthObs = sumIdepthObs / sumIVarObs;
            idepthObs = unzero_f(idepthObs);
            hf = make_float4(idepthObs, VAR_RANDOM_INIT_INITIAL, -1.f, -1.f);
            hi = make_int4(1, 0, 0, __float_as_int(0.f));
        }
    }
    dst.hf[idx] = hf;
    dst.hi[idx] = hi;
}

// regularizeDepthMapRow<removeOcclusions>, DepthMap.cpp:758-848.  dst = src with smoothed values / removals.
template <bool removeOcclusions>
__global__ void __launch_bounds__(256) k_regularize(HypField src, HypField dst, DepthCam cam, DepthGlobals G, int validityTH)
{
    // 32x8 output pixels per CTA; the 36x12 neighbourhood (idepth, var, validity, valid) is staged once in
    // shared memory, so each hypothesis is fetched from L2 1.7x instead of 25x
    __shared__ float4 tile[12][36];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int x0 = blockIdx.x * 32 - 2, y0 = blockIdx.y * 8 - 2;
    const int width = cam.w;
    for (int t = threadIdx.x; t < 12 * 36; t += 256) {
        const int lx = t % 36, ly = t / 36;
        const int gx = x0 + lx, gy = y0 + ly;
        float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gx >= 0 && gx < width && gy >= 0 && gy < cam.h) {
            const int4 si = src.hi[gx + gy * width];
            if (si.x) {
                const float4 s = src.hf[gx + gy * width];
                e = make_float4(s.x, s.y, __int_as_float(si.z), __int_as_float(1));
            }
        }
        tile[ly][lx] = e;
    }
    __syncthreads();
    const int x = blockIdx.x * 32 + tx;
    const int y = blockIdx.y * 8 + ty;
    if (x >= cam.w || y >= cam.h) return;
    const int idx = x + y * width;
    float4 hf = src.hf[idx];
    int4 hi = src.hi[idx];
    if (x >= 2 && x < width - 2 && y >= 2 && y < cam.h - 2 && hi.x) {
        const float regDistVar = G.regDistVar;
        float sum = 0, val_sum = 0, sumIvar = 0;
        int numOccluding = 0, numNotOccluding = 0;
        for (int dx = -2; dx <= 2; dx++)                 // dx outer, dy inner as in the reference (:782-783)
            for (int dy = -2; dy <= 2; dy++) {
                const float4 s = tile[ty + 2 + dy][tx + 2 + dx];
                if (!__float_as_int(s.w)) continue;
                int4 si;
                si.z = __float_as_int(s.z);
                float diff = s.x - hf.x;
                if (DIFF_FAC_SMOOTHING * diff * diff > s.y + hf.y) {
                    if (removeOcclusions) {
                        if (s.x > hf.x) numOccluding++;
                    }
                    continue;
                }
                val_sum += si.z;
                if (removeOcclusions) numNotOccluding++;
                float distFac = (float)(dx * dx + dy * dy) * regDistVar;
                float ivar = 1.0f / (s.y + distFac);
                sum += s.x * ivar;
                sumIvar += ivar;
            }
        if (val_sum < validityTH) {
            hi.x = 0;
            hi.y--;
        } else if (removeOcclusions && numOccluding > numNotOccluding) {
            hi.x = 0;
        } else {
            sum = sum / sumIvar;
            sum = unzero_f(sum);
            hf.z = sum;
            hf.w = 1.0f / sumIvar;
        }
    }
    dst.hf[idx] = hf;
    dst.hi[idx] = hi;
}

// last-CTA-done combine of per-CTA (sum, count) partials in a fixed order; out[0] = sum, out[1] = count,
// out[2] = rescaleFactor = count / sum evaluated in float like DepthMap.cpp:1294
__device__ __forceinline__ void finishSumCount(double s, int c, double* __restrict__ partials, unsigned int* counter,
                                               double* __restrict__ out)
{
    __shared__ double ssum[16];
    __shared__ double scnt[16];
    __shared__ bool isLast;
    const int nWarps = blockDim.x >> 5;
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        c += __shfl_xor_sync(0xffffffffu, c, o);
    }
    if ((threadIdx.x & 31) == 0) { ssum[threadIdx.x >> 5] = s; scnt[threadIdx.x >> 5] = (double)c; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0, tc = 0;
        for (int k = 0; k < nWarps; k++) { t += ssum[k]; tc += scnt[k]; }
        __stcg(partials + 2 * blockIdx.x, t);
        __stcg(partials + 2 * blockIdx.x + 1, tc);
        __threadfence();
        unsigned int tk = atomicAdd(counter, 1u);
        isLast = (tk == gridDim.x - 1);
    }
    __syncthreads();
    if (!isLast) return;
    __threadfence();
    double a = 0, b = 0;
    for (int k = threadIdx.x; k < (int)gridDim.x; k += blockDim.x) { a += __ldcg(partials + 2 * k); b += __ldcg(partials + 2 * k + 1); }
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { ssum[threadIdx.x >> 5] = a; scnt[threadIdx.x >> 5] = b; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double S = 0, Cn = 0;
        for (int k = 0; k < nWarps; k++) { S += ssum[k]; Cn += scnt[k]; }
        out[0] = S; out[1] = Cn;
        out[2] = (double)((float)Cn / (float)S);
        *counter = 0;
    }
}

// regularizeDepthMapFillHoles (DepthMap.cpp:656-718) immediately followed by regularizeDepthMap(false, TH)
// (:758-880) -- the pair that updateKeyframe (:1135-1143), createKeyFrame (:1270-1277) and finalizeKeyFrame
// (:1373-1379) always run back to back -- as ONE kernel, optionally (SETDEPTH) followed in the same kernel by
// Frame::setDepth + Frame::buildIDepthAndIDepthVar (Frame.cpp:199-243, 775-877; updateKeyframe :1150-1157,
// finalizeKeyFrame :1385).  A CTA produces a 32x16 tile: stage 1 stages the 40x24 source neighbourhood in shared
// memory, stage 2 evaluates fill-holes on the 36x20 region the regulariser will look at, stage 3 regularises the tile,
// stage 4 exports idepth / idepthVar of the tile and its 16x8, 8x4, 4x2, 2x1 pyramid blocks and the ordered
// sum / count.  Per-pixel arithmetic and its order are those of the separate kernels, so the result is bit-identical to
// running them one after the other; it saves two launches and two round trips of the 9.8 MB hypothesis planes.
#define FR_TW 32
#define FR_TH 16
#define FR_PPT 2                          // pixels per thread in the regularise stage: all CTAs resident in ONE wave (see DESIGN.md)
#define FR_THREADS (FR_TW * FR_TH / FR_PPT)
template <bool SETDEPTH>
__global__ void __launch_bounds__(FR_THREADS) k_fill_regularize(HypField src, HypField dst, DepthCam cam, DepthGlobals G,
                                                                const float* __restrict__ kfMaxGrad, int validityTH,
                                                                PyrPtrs id, PyrPtrs var, double* __restrict__ partials,
                                                                unsigned int* counter, double* __restrict__ statsOut)
{
    __shared__ float4 sA[FR_TH + 8][FR_TW + 8];      // source:      (idepth, idepth_var, validity_counter, isValid)
    __shared__ float4 sB[FR_TH + 4][FR_TW + 4];      // after fill:  same fields
    __shared__ unsigned char sCreated[FR_TH + 4][FR_TW + 4];
    pdlWait();                                       // launched early (programmatic dependent launch): wait for k_observe
    const int width = cam.w, height = cam.h;
    const int tilesX = (width + FR_TW - 1) / FR_TW;
    const int bx = blockIdx.x % tilesX, by = blockIdx.x / tilesX;
    const int ax0 = bx * FR_TW - 4, ay0 = by * FR_TH - 4;
    for (int t = threadIdx.x; t < (FR_TH + 8) * (FR_TW + 8); t += FR_THREADS) {
        const int lx = t % (FR_TW + 8), ly = t / (FR_TW + 8);
        const int gx = ax0 + lx, gy = ay0 + ly;
        float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gx >= 0 && gx < width && gy >= 0 && gy < height) {
            const int4 si = src.hi[gx + gy * width];
            if (si.x) {
                const float4 sf = src.hf[gx + gy * width];
                e = make_float4(sf.x, sf.y, __int_as_float(si.z), __int_as_float(1));
            }
        }
        sA[ly][lx] = e;
    }
    __syncthreads();
    // stage 2: fill holes on the region the regulariser reads (tile + 2)
    for (int t = threadIdx.x; t < (FR_TH + 4) * (FR_TW + 4); t += FR_THREADS) {
        const int lx = t % (FR_TW + 4), ly = t / (FR_TW + 4);
        const int gx = ax0 + 2 + lx, gy = ay0 + 2 + ly;
        float4 e = sA[ly + 2][lx + 2];
        unsigned char created = 0;
        if (gx >= 3 && gx < width - 2 && gy >= 3 && gy < height - 2 && !__float_as_int(e.w)) {
            const int idx = gx + gy * width;
            if (!(kfMaxGrad[idx] < G.minUseGrad)) {
                int val = 0;
                for (int dy = -2; dy <= 2; dy++)
                    for (int dx = -2; dx <= 2; dx++) {
                        const float4 q = sA[ly + 2 + dy][lx + 2 + dx];
                        if (__float_as_int(q.w)) val += __float_as_int(q.z);
                    }
                const int blacklisted = src.hi[idx].y;
                if ((blacklisted >= MIN_BLACKLIST && val > VAL_SUM_MIN_FOR_CREATE) || val > VAL_SUM_MIN_FOR_UNBLACKLIST) {
                    float sumIdepthObs = 0, sumIVarObs = 0;
                    for (int dy = -2; dy <= 2; dy++)         // row-major source order, :679-688
                        for (int dx = -2; dx <= 2; dx++) {
                            const float4 q = sA[ly + 2 + dy][lx + 2 + dx];
                            if (!__float_as_int(q.w)) continue;
                            sumIdepthObs += q.x / q.y;
                            sumIVarObs += 1.0f / q.y;
                        }
                    float idepthObs = sumIdepthObs / sumIVarObs;
                    idepthObs = unzero_f(idepthObs);
                    e = make_float4(idepthObs, VAR_RANDOM_INIT_INITIAL, __int_as_float(0), __int_as_float(1));
                    created = 1;
                }
            }
        }
        sB[ly][lx] = e;
        sCreated[ly][lx] = created;
    }
    __syncthreads();
    // stage 3: regularizeDepthMapRow<false> on the tile; a thread owns the pixels (tx, ty) and (tx, ty + FR_TH/2)
    const int tx = threadIdx.x % FR_TW, ty0 = threadIdx.x / FR_TW;
    float2 vOut[FR_PPT];
    double ssum = 0.0;
    int scnt = 0;
#pragma unroll
    for (int pp = 0; pp < FR_PPT; pp++) {
        const int ty = ty0 + pp * (FR_TH / FR_PPT);
        const int x = bx * FR_TW + tx, y = by * FR_TH + ty;
        const bool inside = x < width && y < height;
        const int idx = x + y * width;
        float4 hf = make_float4(0.f, 0.f, 0.f, 0.f);
        int4 hi = make_int4(0, 0, 0, 0);
        if (inside) {
            if (sCreated[ty + 2][tx + 2]) {  // fresh DepthMapPixelHypothesis(idepth, var, 0): blacklisted = 0, smoothed = -1
                const float4 c = sB[ty + 2][tx + 2];
                hf = make_float4(c.x, c.y, -1.f, -1.f);
                hi = make_int4(1, 0, 0, __float_as_int(0.f));
            } else {
                hf = src.hf[idx];
                hi = src.hi[idx];
            }
            if (x >= 2 && x < width - 2 && y >= 2 && y < height - 2 && hi.x) {
                const float regDistVar = G.regDistVar;
                float sum = 0, val_sum = 0, sumIvar = 0;
                for (int dx = -2; dx <= 2; dx++)             // dx outer, dy inner as in the reference (:782-783)
                    for (int dy = -2; dy <= 2; dy++) {
                        const float4 q = sB[ty + 2 + dy][tx + 2 + dx];
                        if (!__float_as_int(q.w)) continue;
                        const float diff = q.x - hf.x;
                        if (DIFF_FAC_SMOOTHING * diff * diff > q.y + hf.y) continue;
                        val_sum += __float_as_int(q.z);
                        const float distFac = (float)(dx * dx + dy * dy) * regDistVar;
                        const float ivar = 1.0f / (q.y + distFac);
                        sum += q.x * ivar;
                        sumIvar += ivar;
                    }
                if (val_sum < validityTH) {
                    hi.x = 0;
                    hi.y--;
                } else {
                    sum = sum / sumIvar;
                    sum = unzero_f(sum);
                    hf.z = sum;
                    hf.w = 1.0f / sumIvar;
                }
            }
            dst.hf[idx] = hf;
            dst.hi[idx] = hi;
        }
        if (SETDEPTH) {
            // Frame::setDepth (Frame.cpp:217-232): level-0 idepth / idepthVar and the frame's sum / count
            float2 v = make_float2(-1.f, -1.f);
            if (inside && hi.x && hf.z >= -0.05) { v = make_float2(hf.z, hf.w); ssum += (double)hf.z; scnt++; }
            if (inside) { id.l[0][idx] = v.x; var.l[0][idx] = v.y; }
            vOut[pp] = v;
        }
    }
    if (!SETDEPTH) return;
    // stage 4: idepth pyramid blocks of this tile (Frame::buildIDepthAndIDepthVar, Frame.cpp:775-877) + ordered sum / count
    float2* t0 = reinterpret_cast<float2*>(&sA[0][0]);          // sA is dead: reuse it for the pyramid staging
    float2* t1 = t0 + FR_TW * FR_TH;
    float2* t2 = t1 + (FR_TW / 2) * (FR_TH / 2);
    float2* t3 = t2 + (FR_TW / 4) * (FR_TH / 4);
    __syncthreads();
#pragma unroll
    for (int pp = 0; pp < FR_PPT; pp++) t0[(ty0 + pp * (FR_TH / FR_PPT)) * FR_TW + tx] = vOut[pp];
    __syncthreads();
    {
        const int t = threadIdx.x;                               // (FR_TW/2) x (FR_TH/2) = 128 outputs
        if (t < (FR_TW / 2) * (FR_TH / 2)) {
            const int px = t % (FR_TW / 2), py = t / (FR_TW / 2);
            const float2 r = mergeIdepth4(t0[(2 * py) * FR_TW + 2 * px], t0[(2 * py) * FR_TW + 2 * px + 1],
                                          t0[(2 * py + 1) * FR_TW + 2 * px], t0[(2 * py + 1) * FR_TW + 2 * px + 1]);
            t1[py * (FR_TW / 2) + px] = r;
            const int ox = bx * (FR_TW / 2) + px, oy = by * (FR_TH / 2) + py;
            if (ox < (width >> 1) && oy < (height >> 1)) { id.l[1][oy * (width >> 1) + ox] = r.x; var.l[1][oy * (width >> 1) + ox] = r.y; }
        }
    }
    __syncthreads();
    {
        const int t = threadIdx.x;
        if (t < (FR_TW / 4) * (FR_TH / 4)) {
            const int W1 = FR_TW / 2;
            const int px = t % (FR_TW / 4), py = t / (FR_TW / 4);
            const float2 r = mergeIdepth4(t1[(2 * py) * W1 + 2 * px], t1[(2 * py) * W1 + 2 * px + 1],
                                          t1[(2 * py + 1) * W1 + 2 * px], t1[(2 * py + 1) * W1 + 2 * px + 1]);
            t2[py * (FR_TW / 4) + px] = r;
            const int ox = bx * (FR_TW / 4) + px, oy = by * (FR_TH / 4) + py;
            if (ox < (width >> 2) && oy < (height >> 2)) { id.l[2][oy * (width >> 2) + ox] = r.x; var.l[2][oy * (width >> 2) + ox] = r.y; }
        }
    }
    __syncthreads();
    {
        const int t = threadIdx.x;
        if (t < (FR_TW / 8) * (FR_TH / 8)) {
            const int W2 = FR_TW / 4;
            const int px = t % (FR_TW / 8), py = t / (FR_TW / 8);
            const float2 r = mergeIdepth4(t2[(2 * py) * W2 + 2 * px], t2[(2 * py) * W2 + 2 * px + 1],
                                          t2[(2 * py + 1) * W2 + 2 * px], t2[(2 * py + 1) * W2 + 2 * px + 1]);
            t3[py * (FR_TW / 8) + px] = r;
            const int ox = bx * (FR_TW / 8) + px, oy = by * (FR_TH / 8) + py;
            if (ox < (width >> 3) && oy < (height >> 3)) { id.l[3][oy * (width >> 3) + ox] = r.x; var.l[3][oy * (width >> 3) + ox] = r.y; }
        }
    }
    __syncthreads();
    {
        const int t = threadIdx.x;
        if (t < (FR_TW / 16) * (FR_TH / 16)) {
            const int W3 = FR_TW / 8;
            const int px = t % (FR_TW / 16), py = t / (FR_TW / 16);
            const float2 r = mergeIdepth4(t3[(2 * py) * W3 + 2 * px], t3[(2 * py) * W3 + 2 * px + 1],
                                          t3[(2 * py + 1) * W3 + 2 * px], t3[(2 * py + 1) * W3 + 2 * px + 1]);
            const int ox = bx * (FR_TW / 16) + px, oy = by * (FR_TH / 16) + py;
            if (ox < (width >> 4) && oy < (height >> 4)) { id.l[4][oy * (width >> 4) + ox] = r.x; var.l[4][oy * (width >> 4) + ox] = r.y; }
        }
    }
    finishSumCount(ssum, scnt, partials, counter, statsOut);
}

// Frame::setDepth fused with Frame::buildIDepthAndIDepthVar for levels 1..4 (Frame.cpp:199-243 + :775-877): one CTA =
// one 16x16 level-0 tile; the tracker imports the new depth right after every update, so the pyramid is always
// needed and building it here saves a pass over the level-0 planes and a launch.
__global__ void __launch_bounds__(256) k_set_depth_pyr(HypField cur, PyrPtrs id, PyrPtrs var, int w, int h,
                                                       double* __restrict__ partials, unsigned int* counter, double* __restrict__ out)
{
    __shared__ float2 s0[16][17], s1[8][9], s2[4][5], s3[2][3];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int tilesX = w >> 4;
    const int bx = blockIdx.x % tilesX, by = blockIdx.x / tilesX;
    const int x = bx * 16 + tx, y = by * 16 + ty;
    const int i = x + y * w;
    double s = 0.0;
    int c = 0;
    float2 v;
    {
        const float4 hf = cur.hf[i];
        const int4 hi = cur.hi[i];
        if (hi.x && hf.z >= -0.05) { v = make_float2(hf.z, hf.w); s = hf.z; c = 1; }
        else v = make_float2(-1.f, -1.f);
    }
    id.l[0][i] = v.x; var.l[0][i] = v.y;
    s0[ty][tx] = v;
    __syncthreads();
    if (tx < 8 && ty < 8) {
        float2 r = mergeIdepth4(s0[2 * ty][2 * tx], s0[2 * ty][2 * tx + 1], s0[2 * ty + 1][2 * tx], s0[2 * ty + 1][2 * tx + 1]);
        s1[ty][tx] = r;
        int o = (by * 8 + ty) * (w >> 1) + bx * 8 + tx;
        id.l[1][o] = r.x; var.l[1][o] = r.y;
    }
    __syncthreads();
    if (tx < 4 && ty < 4) {
        float2 r = mergeIdepth4(s1[2 * ty][2 * tx], s1[2 * ty][2 * tx + 1], s1[2 * ty + 1][2 * tx], s1[2 * ty + 1][2 * tx + 1]);
        s2[ty][tx] = r;
        int o = (by * 4 + ty) * (w >> 2) + bx * 4 + tx;
        id.l[2][o] = r.x; var.l[2][o] = r.y;
    }
    __syncthreads();
    if (tx < 2 && ty < 2) {
        float2 r = mergeIdepth4(s2[2 * ty][2 * tx], s2[2 * ty][2 * tx + 1], s2[2 * ty + 1][2 * tx], s2[2 * ty + 1][2 * tx + 1]);
        s3[ty][tx] = r;
        int o = (by * 2 + ty) * (w >> 3) + bx * 2 + tx;
        id.l[3][o] = r.x; var.l[3][o] = r.y;
    }
    __syncthreads();
    if (tx == 0 && ty == 0) {
        float2 r = mergeIdepth4(s3[0][0], s3[0][1], s3[1][0], s3[1][1]);
        int o = by * (w >> 4) + bx;
        id.l[4][o] = r.x; var.l[4][o] = r.y;
    }
    finishSumCount(s, c, partials, counter, out);
}

// createKeyFrame :1295-1304
__global__ void __launch_bounds__(256) k_rescale(HypField cur, int n, const double* __restrict__ scal)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!cur.hi[i].x) return;
    const float rescaleFactor = (float)scal[2];
    const float rescaleFactor2 = rescaleFactor * rescaleFactor;
    float4 hf = cur.hf[i];
    hf.x *= rescaleFactor; hf.z *= rescaleFactor; hf.y *= rescaleFactor2; hf.w *= rescaleFactor2;
    cur.hf[i] = hf;
}

// ---------------------------------------------------------------------------------------------------------
// propagateDepth, DepthMap.cpp:475-653.  The reference is a serial raster scan whose result depends on the
// ORDER in which sources hit a target.  Phase 1 projects every source and threads it onto a per-target list;
// phase 2 (one thread per target) replays its sources in ascending source index == raster order.
// ---------------------------------------------------------------------------------------------------------
struct PropParams {
    float R[9], t[3];
    const uint8_t* trackingWasGood;   // new keyframe's refPixelWasGood (or nullptr)
    const float* activeKFImage;
    const float* newKFMaxGrad;
    const float* newKFImage;
};
__global__ void __launch_bounds__(256) k_prop_project(HypField src, DepthCam cam, DepthGlobals G, PropParams P,
                                                      int* __restrict__ head, int* __restrict__ next, float4* __restrict__ val)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int width = cam.w, height = cam.h;
    if (i >= width * height) return;
    int4 hi = src.hi[i];
    if (!hi.x) return;
    const int x = i % width, y = i / width;
    float4 hf = src.hf[i];
    float p0 = x * cam.fxi + cam.cxi, p1 = y * cam.fyi + cam.cyi, p2 = 1.0f;
    float pn0 = ((P.R[0] * p0 + P.R[1] * p1) + P.R[2] * p2) / hf.z + P.t[0];
    float pn1 = ((P.R[3] * p0 + P.R[4] * p1) + P.R[5] * p2) / hf.z + P.t[1];
    float pn2 = ((P.R[6] * p0 + P.R[7] * p1) + P.R[8] * p2) / hf.z + P.t[2];
    float new_idepth = 1.0f / pn2;
    float u_new = pn0 * new_idepth * cam.fx + cam.cx;
    float v_new = pn1 * new_idepth * cam.fy + cam.cy;
    if (!(u_new > 2.1f && v_new > 2.1f && u_new < width - 3.1f && v_new < height - 3.1f)) return;
    int newIDX = (int)(u_new + 0.5f) + ((int)(v_new + 0.5f)) * width;
    float destAbsGrad = P.newKFMaxGrad[newIDX];
    if (P.trackingWasGood != nullptr) {
        if (!P.trackingWasGood[(x >> SE3TRACKING_MIN_LEVEL) + (width >> SE3TRACKING_MIN_LEVEL) * (y >> SE3TRACKING_MIN_LEVEL)]
            || destAbsGrad < G.minUseGrad)
            return;
    } else {
        float sourceColor = P.activeKFImage[i];
        float destColor = interpF(P.newKFImage, u_new, v_new, width);
        float residual = destColor - sourceColor;
        if (residual * residual / (MAX_DIFF_CONSTANT + MAX_DIFF_GRAD_MULT * destAbsGrad * destAbsGrad) > 1.0f || destAbsGrad < G.minUseGrad)
            return;
    }
    float idepth_ratio_4 = new_idepth / hf.z;
    idepth_ratio_4 *= idepth_ratio_4;
    idepth_ratio_4 *= idepth_ratio_4;
    float new_var = idepth_ratio_4 * hf.y;
    val[i] = make_float4(new_idepth, new_var, __int_as_float(hi.z), 0.f);
    next[i] = atomicExch(head + newIDX, i);
}
__global__ void __launch_bounds__(256) k_prop_resolve(HypField dst, int n, const int* __restrict__ head,
                                                      const int* __restrict__ next, const float4* __restrict__ val)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Hyp t;
    t.isValid = 0; t.blacklisted = 0; t.validity_counter = 0; t.nextStereoFrameMinID = 0;      // :496-500
    t.idepth = 0; t.idepth_var = 0; t.idepth_smoothed = 0; t.idepth_var_smoothed = 0;
    const int h0 = head[i];
    int last = -1;
    while (h0 >= 0) {
        // next source in raster order: the smallest list entry larger than `last`
        int best = 0x7fffffff;
        for (int s = h0; s >= 0; s = next[s])
            if (s > last && s < best) best = s;
        if (best == 0x7fffffff) break;
        last = best;
        const float4 sv = val[best];
        const float new_idepth = sv.x, new_var = sv.y;
        const int src_validity = __float_as_int(sv.z);
        bool skip = false;
        if (t.isValid) {                                                         // :584-603
            float diff = t.idepth - new_idepth;
            if (DIFF_FAC_PROP_MERGE * diff * diff > new_var + t.idepth_var) {
                if (new_idepth < t.idepth) skip = true;
                else t.isValid = 0;
            }
        }
        if (skip) continue;
        if (!t.isValid) {
            hypCtor3(t, new_idepth, new_var, src_validity);                      // :606-615
        } else {
            float w = new_var / (t.idepth_var + new_var);                        // :616-633
            float merged_new_idepth = w * t.idepth + (1.0f - w) * new_idepth;
            int merged_validity = src_validity + t.validity_counter;
            if (merged_validity > VALIDITY_COUNTER_MAX + (VALIDITY_COUNTER_MAX_VARIABLE))
                merged_validity = VALIDITY_COUNTER_MAX + (VALIDITY_COUNTER_MAX_VARIABLE);
            float mv = 1.0f / (1.0f / t.idepth_var + 1.0f / new_var);
            hypCtor3(t, merged_new_idepth, mv, merged_validity);
        }
    }
    storeHyp(dst, i, t);
}

// initializeFromGTDepth, DepthMap.cpp:993-1014: hypotheses from the keyframe's level-0 idepth
__global__ void __launch_bounds__(256) k_init_from_gt(HypField cur, const float* __restrict__ idepth, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v = idepth[i];
    int4 hi = cur.hi[i];
    float4 hf = cur.hf[i];
    if (!isnan(v) && v > 0) {
        hf = make_float4(v, 0.01f * 0.01f, v, 0.01f * 0.01f);
        hi = make_int4(1, 0, 20, __float_as_int(0.f));
    } else {
        hi.x = 0;
        hi.y = 0;
    }
    cur.hf[i] = hf;
    cur.hi[i] = hi;
}

// AoS (reference layout) <-> the two 16-byte planes.  aos is 16-byte aligned (the staging buffer, or a caller's buffer checked by
// lsdgpu_depth_set_hypotheses_device / lsdgpu_depth_download_device), so a 32-byte record moves as two 128-bit accesses: the
// words {isValid + pad, blacklisted, nextStereoFrameMinID, validity_counter}, then the four idepth floats.
__global__ void __launch_bounds__(256) k_hyp_from_aos(const lsdgpu_hyp* __restrict__ aos, HypField f, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int4* rec = reinterpret_cast<const int4*>(aos + i);
    const int4 a = __ldg(rec);
    const float4 b = __ldg(reinterpret_cast<const float4*>(rec + 1));
    f.hf[i] = b;
    f.hi[i] = make_int4((a.x & 0xff) ? 1 : 0, a.y, a.w, a.z);     // isValid is the low byte of word 0 (little endian)
}
__global__ void __launch_bounds__(256) k_hyp_to_aos(HypField f, lsdgpu_hyp* __restrict__ aos, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 a = f.hf[i];
    const int4 b = f.hi[i];
    int4* rec = reinterpret_cast<int4*>(aos + i);
    rec[0] = make_int4(b.x ? 1 : 0, b.y, b.w, b.z);              // isValid as 0 / 1 with its three pad bytes 0
    *reinterpret_cast<float4*>(rec + 1) = a;
}

// validityIntegralBuffer on demand (parity hook only; the hot path never builds it), DepthMap.cpp:722-754
__global__ void k_integral_rows(HypField cur, int* __restrict__ integral, int w, int h)
{
    const int y = blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= h) return;
    int s = 0;
    for (int x = 0; x < w; x++) {
        int4 hi = cur.hi[y * w + x];
        if (hi.x) s += hi.z;
        integral[y * w + x] = s;
    }
}
__global__ void k_integral_cols(int* __restrict__ integral, int w, int h)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= w) return;
    int s = integral[x];
    for (int y = 1; y < h; y++) {
        s += integral[y * w + x];
        integral[y * w + x] = s;
    }
}

// Frame::takeReActivationData: entries of invalid pixels keep idepth / validity (only the variance code is written)
__global__ void __launch_bounds__(256) k_take_reactivation(HypField cur, float* __restrict__ idepthReAct, float* __restrict__ varReAct,
                                                           uint8_t* __restrict__ validityReAct, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int4 hi = cur.hi[i];
    if (hi.x) {
        const float4 hf = cur.hf[i];
        idepthReAct[i] = hf.x;
        varReAct[i] = hf.y;
        validityReAct[i] = (uint8_t)hi.z;
    } else if (hi.y < -1)                       // blacklisted < MIN_BLACKLIST (util/settings.h:117)
        varReAct[i] = -2;
    else
        varReAct[i] = -1;
}

// DepthMap::setFromExistingKF: DepthMapPixelHypothesis(idepth, idepth_var, validity) (DepthMapPixelHypothesis.h:80-91) or
// invalid with the blacklist code; fields the reference leaves untouched on invalid pixels are left untouched here too
__global__ void __launch_bounds__(256) k_set_from_existing(const float* __restrict__ idepthReAct, const float* __restrict__ varReAct,
                                                           const uint8_t* __restrict__ validityReAct, HypField cur, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float var = varReAct[i];
    if (var > 0) {
        cur.hf[i] = make_float4(idepthReAct[i], var, -1.f, -1.f);
        cur.hi[i] = make_int4(1, 0, (int)validityReAct[i], 0);
    } else {
        int4 hi = cur.hi[i];
        hi.x = 0;
        hi.y = (var == -2) ? -2 : 0;            // MIN_BLACKLIST - 1
        cur.hi[i] = hi;
    }
}
