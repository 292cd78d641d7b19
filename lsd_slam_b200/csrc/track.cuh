// track.cuh -- the fused warp / residual / weight / Jacobian / normal-equation evaluation of SE3Tracker (device code; the
// stand-alone evaluation kernel k_se3_eval is in tracking.cu, the persistent tracker in track_persistent.cuh).
//
// Replaces (paths relative to lsd_slam_core/src/):
//   TrackingReference::makePointCloud     Tracking/TrackingReference.cpp:96-147   (never materialised: each
//                                         thread rebuilds its point from the keyframe's idepth pyramid)
//   SE3Tracker::calcResidualAndBuffers    Tracking/SE3Tracker.cpp:885-1029        (hot loop A)
//   SE3Tracker::calcWeightsAndResidual    Tracking/SE3Tracker.cpp:749-790         (hot loop B, scalar semantics)
//   SE3Tracker::calculateWarpUpdate       Tracking/SE3Tracker.cpp:1258-1299       (hot loop C)
//   LGS6::update / finish                 Tracking/LGSX.h:390-396, 319-325
//
// Mapping: DENSE, one thread per keyframe pixel of the level (x fastest), so the three keyframe planes
// (idepth, idepthVar, colour) are read fully coalesced and the four bilinear taps of neighbouring threads
// land on neighbouring float4 texels of the new frame's gradient level.  Nothing is written per point except
// the level-1 refPixelWasGood byte; the 8 SoA buffers of the reference never exist.  Each CTA reduces
// EV_NCH channels with warp shuffles + one shared-memory stage, writes one partial row, and the LAST CTA to
// finish sums the rows in block order (deterministic, no float atomics) in double.
#pragma once
#include "internal.cuh"

// reduction channels
enum {
    CH_A = 0,        // 21 upper-triangle entries of sum J J^T w, row-major (i <= j)
    CH_B = 21,       // 6: sum J r w        (LGS6::b = -this)
    CH_SUMRESW = 27, // sum wh w_p r r      (calcWeightsAndResidual; LGS6::error is the same sum, LGSX.h:394)
    CH_SUMRESU = 28, // sum r r over good   (sumResUnweighted)
    CH_SIGNED = 29,  // sum r over good     (sumSignedRes)
    CH_GOOD = 30, CH_BAD = 31,              // buf_warped_size == good + bad (exact: integer-valued floats)
    CH_USAGE = 32,
    CH_REFNUM = 33,  // numData[level]
    CH_SXX = 34, CH_SYY = 35, CH_SX = 36, CH_SY = 37, CH_SW = 38      // 39: unused (pads to 32 + 8)
};

struct EvalLevel {
    const float* __restrict__ kfIdepth;
    const float* __restrict__ kfVar;
    const float* __restrict__ kfColor;
    const float4* __restrict__ frameGrad;
    uint8_t* goodMask;              // level-1 mask or nullptr
    int w, h;
    float fx, fy, cx, cy, fxi, fyi, cxi, cyi;
    int shard, nShards;             // point sharding across GPUs: this rank owns 32-px chunks c with c % nShards == shard
};
struct EvalPose {
    float R[9], t[3];
    float a, b;                     // affineEstimation_a / _b
};
struct EvalConsts {
    float cameraPixelNoise2, var_weight, huber_half;
};

// Rows 3 and 4 of the Jacobian carry double literals in the reference (SE3Tracker.cpp:1284-1285):
//     v[3] = (-Wx*Wy*z_sqr)*gx + (-(1.0 + Wy*Wy*z_sqr))*gy          -> (float)((double)a + (-(1.0 + (double)b)) * (double)g)
// i.e. the float nearest to  a - g - b*g  (a, b, g floats), computed through two 53-bit roundings.  FP64 issues at half
// the FP32 rate on H100 and this sits on the per-point path of every evaluation, so the value is
// formed from error-free float transformations instead: b*g = ph + pl exactly (FMA), two TwoSums carry the rounding errors
// of a - g - ph, and one last add rounds once.  The result is the correctly rounded float of the exact expression; it can
// differ from the reference's doubly rounded one only when the exact value lies within 2^-29 ulp of a rounding boundary
// (about once in 10^8 points, one ulp of one Jacobian entry).
__device__ __forceinline__ float jacRowMixed(float a, float b, float g)
{
    const float ph = b * g;
    const float pl = fmaf(b, g, -ph);
    const float s = a - g;
    const float sv = s - a;
    const float se = (a - (s - sv)) + (-g - sv);
    const float t = s - ph;
    const float tv = t - s;
    const float te = (s - (t - tv)) + (-ph - tv);
    return t + ((se + te) - pl);
}

struct PointAcc {
    float v[EV_NCH];
};

// getInterpolatedElement43, util/globalFuncs.h:63-77 (weights and summation order of the reference)
__device__ __forceinline__ void interp43(const float4* __restrict__ mat, float x, float y, int width, float& o0, float& o1, float& o2)
{
    int ix = (int)x, iy = (int)y;
    float dx = x - ix, dy = y - iy;
    float dxdy = dx * dy;
    const float4* bp = mat + ix + iy * width;
    float4 br = __ldg(bp + 1 + width), bl = __ldg(bp + width), tr = __ldg(bp + 1), tl = __ldg(bp);
    float w0 = dxdy, w1 = (dy - dxdy), w2 = (dx - dxdy), w3 = (1 - dx - dy + dxdy);
    o0 = w0 * br.x + w1 * bl.x + w2 * tr.x + w3 * tl.x;
    o1 = w0 * br.y + w1 * bl.y + w2 * tr.y + w3 * tl.y;
    o2 = w0 * br.z + w1 * bl.z + w2 * tr.z + w3 * tl.z;
}

// One keyframe pixel -> its contribution to all channels.  `valid` = the makePointCloud test
// (TrackingReference.cpp:128-133).  Returns the refPixelWasGood value to store (0/1), or -1 if none.
template <typename TapFn>
__device__ __forceinline__ int evalPoint(float px, float py, float pz, float color, float var,
                                         const EvalPose& P, const EvalConsts& C,
                                         float fx_l, float fy_l, float cx_l, float cy_l, int w, int h,
                                         TapFn tap, PointAcc& acc)
{
    // SE3Tracker.cpp:937-939
    float Wx = ((P.R[0] * px + P.R[1] * py) + P.R[2] * pz) + P.t[0];
    float Wy = ((P.R[3] * px + P.R[4] * py) + P.R[5] * pz) + P.t[1];
    float Wz = ((P.R[6] * px + P.R[7] * py) + P.R[8] * pz) + P.t[2];
    float u_new = (Wx / Wz) * fx_l + cx_l;
    float v_new = (Wy / Wz) * fy_l + cy_l;
    acc.v[CH_REFNUM] += 1.f;
    if (!(u_new > 1 && v_new > 1 && u_new < w - 2 && v_new < h - 2)) return 0;   // :943-948

    float gi0, gi1, gi2;
    tap(u_new, v_new, gi0, gi1, gi2);                                              // :950

    float c1 = P.a * color + P.b;                                                 // :952-954
    float c2 = gi2;
    float residual = c1 - c2;
    float weight = fabsf(residual) < 5.0f ? 1 : 5.0f / fabsf(residual);           // :956-961
    acc.v[CH_SXX] += c1 * c1 * weight;
    acc.v[CH_SYY] += c2 * c2 * weight;
    acc.v[CH_SX] += c1 * weight;
    acc.v[CH_SY] += c2 * weight;
    acc.v[CH_SW] += weight;
    bool isGood = residual * residual / ((40.0f * 40.0f) + (0.5f * 0.5f) * (gi0 * gi0 + gi1 * gi1)) < 1;   // :963

    float gx = fx_l * gi0, gy = fy_l * gi1;                                       // :972-973
    float d = 1.0f / pz;                                                          // :976
    if (isGood) {                                                                 // :981-988
        acc.v[CH_SUMRESU] += residual * residual;
        acc.v[CH_SIGNED] += residual;
        acc.v[CH_GOOD] += 1.f;
    } else
        acc.v[CH_BAD] += 1.f;
    float depthChange = pz / Wz;                                                  // :990-991
    acc.v[CH_USAGE] += depthChange < 1 ? depthChange : 1;

    // calcWeightsAndResidual, :767-786
    float s = C.var_weight * var;
    float g0 = (P.t[0] * Wz - P.t[2] * Wx) / (Wz * Wz * d);
    float g1 = (P.t[1] * Wz - P.t[2] * Wy) / (Wz * Wz * d);
    float drpdd = gx * g0 + gy * g1;
    float w_p = 1.0f / ((C.cameraPixelNoise2) + s * drpdd * drpdd);
    float weighted_rp = fabsf(residual * sqrtf(w_p));
    float wh = fabsf(weighted_rp < C.huber_half ? 1 : C.huber_half / weighted_rp);
    acc.v[CH_SUMRESW] += wh * w_p * residual * residual;
    float wgt = wh * w_p;

    // calculateWarpUpdate, :1276-1291 (rows 3 and 4 carry double literals in the reference)
    float z = 1.0f / Wz;
    float z_sqr = 1.0f / (Wz * Wz);
    float J[6];
    J[0] = z * gx + 0;
    J[1] = 0 + z * gy;
    J[2] = (-Wx * z_sqr) * gx + (-Wy * z_sqr) * gy;
    J[3] = jacRowMixed((-Wx * Wy * z_sqr) * gx, Wy * Wy * z_sqr, gy);
    J[4] = -jacRowMixed(-((Wx * Wy * z_sqr) * gy), Wx * Wx * z_sqr, gx);
    J[5] = (-Wy * z) * gx + (Wx * z) * gy;

    // LGS6::update, LGSX.h:390-396
    int k = 0;
#pragma unroll
    for (int i = 0; i < 6; i++)
#pragma unroll
        for (int j = i; j < 6; j++) acc.v[CH_A + (k++)] += J[i] * J[j] * wgt;
    float rw = residual * wgt;
#pragma unroll
    for (int i = 0; i < 6; i++) acc.v[CH_B + i] += J[i] * rw;
    return isGood ? 1 : 0;
}

// ---- speculative candidates of the persistent tracker (track_persistent.cuh) -------------------------------------------
// A pass evaluates up to three poses of one LM iteration: the try itself (evalPoint: all channels) and the next one or two
// tries the reference would make IF it rejects (same normal equations, larger lambda, SE3Tracker.cpp:424-447).  Those only
// need what the accept test and the bookkeeping read: the weighted error and the warped-point count -- and, for the last
// candidate of the chain (the pose the level usually ends on), the statistics SlamSystem reads after trackFrame.
// Channel layout of the 16-float extension block:
enum {
    XL_SUMRESW = 0, XL_SUMRESU = 1, XL_SIGNED = 2, XL_GOOD = 3, XL_BAD = 4, XL_USAGE = 5,
    XL_SXX = 6, XL_SYY = 7, XL_SX = 8, XL_SY = 9, XL_SW = 10,           // last candidate: 11 channels
    XM_SUMRESW = 11, XM_GOOD = 12, XM_BAD = 13                          // middle candidate: 3 channels (14, 15: unused)
};
#define EV_NX 16                     // extension channels
#define EV_NCHX (EV_NCH + EV_NX)     // channels of a pass with more than one candidate

// evalPoint without the Jacobian and the normal equations: identical arithmetic for every quantity it accumulates, so that the
// error of a pose evaluated here equals, bit for bit, the error evalPoint gives for the same pose (same reduction tree).
// STATS: also the statistics and affine-lighting sums (last candidate); otherwise error + good / bad counts only.
template <bool STATS, typename TapFn>
__device__ __forceinline__ int evalPointLight(float px, float py, float pz, float color, float var,
                                              const EvalPose& P, const EvalConsts& C,
                                              float fx_l, float fy_l, float cx_l, float cy_l, int w, int h,
                                              TapFn tap, float* x)
{
    float Wx = ((P.R[0] * px + P.R[1] * py) + P.R[2] * pz) + P.t[0];
    float Wy = ((P.R[3] * px + P.R[4] * py) + P.R[5] * pz) + P.t[1];
    float Wz = ((P.R[6] * px + P.R[7] * py) + P.R[8] * pz) + P.t[2];
    float u_new = (Wx / Wz) * fx_l + cx_l;
    float v_new = (Wy / Wz) * fy_l + cy_l;
    if (!(u_new > 1 && v_new > 1 && u_new < w - 2 && v_new < h - 2)) return 0;

    float gi0, gi1, gi2;
    tap(u_new, v_new, gi0, gi1, gi2);

    float c1 = P.a * color + P.b;
    float c2 = gi2;
    float residual = c1 - c2;
    if (STATS) {
        float weight = fabsf(residual) < 5.0f ? 1 : 5.0f / fabsf(residual);
        x[XL_SXX] += c1 * c1 * weight;
        x[XL_SYY] += c2 * c2 * weight;
        x[XL_SX] += c1 * weight;
        x[XL_SY] += c2 * weight;
        x[XL_SW] += weight;
    }
    bool isGood = residual * residual / ((40.0f * 40.0f) + (0.5f * 0.5f) * (gi0 * gi0 + gi1 * gi1)) < 1;

    float gx = fx_l * gi0, gy = fy_l * gi1;
    float d = 1.0f / pz;
    if (STATS) {
        if (isGood) {
            x[XL_SUMRESU] += residual * residual;
            x[XL_SIGNED] += residual;
            x[XL_GOOD] += 1.f;
        } else
            x[XL_BAD] += 1.f;
        float depthChange = pz / Wz;
        x[XL_USAGE] += depthChange < 1 ? depthChange : 1;
    } else {
        if (isGood) x[XM_GOOD] += 1.f;
        else x[XM_BAD] += 1.f;
    }

    float s = C.var_weight * var;
    float g0 = (P.t[0] * Wz - P.t[2] * Wx) / (Wz * Wz * d);
    float g1 = (P.t[1] * Wz - P.t[2] * Wy) / (Wz * Wz * d);
    float drpdd = gx * g0 + gy * g1;
    float w_p = 1.0f / ((C.cameraPixelNoise2) + s * drpdd * drpdd);
    float weighted_rp = fabsf(residual * sqrtf(w_p));
    float wh = fabsf(weighted_rp < C.huber_half ? 1 : C.huber_half / weighted_rp);
    x[STATS ? XL_SUMRESW : XM_SUMRESW] += wh * w_p * residual * residual;
    return isGood ? 1 : 0;
}

#define EVAL_THREADS 256                 // threads per CTA of k_se3_eval (tracking.cu)

// ---- host-side interpretation of the EV_NCH sums (shared by mode 0, the parity hook and mode 1) ----------
LSD_HD void evalFinish(const float* s, lsdgpu_eval_result* r)
{
    static const unsigned char ij[21][2] = { {0,0},{0,1},{0,2},{0,3},{0,4},{0,5},{1,1},{1,2},{1,3},{1,4},{1,5},
                                            {2,2},{2,3},{2,4},{2,5},{3,3},{3,4},{3,5},{4,4},{4,5},{5,5} };
    const float n = s[CH_GOOD] + s[CH_BAD];               // buf_warped_size
    for (int k = 0; k < 21; k++) {
        float a = s[CH_A + k] / n;                         // LGS6::finish, LGSX.h:319-325
        r->A[ij[k][0] * 6 + ij[k][1]] = a;
        r->A[ij[k][1] * 6 + ij[k][0]] = a;
    }
    for (int k = 0; k < 6; k++) r->b[k] = -s[CH_B + k] / n;
    r->lsError = s[CH_SUMRESW] / n;                       // LGS6::error: same sum as calcWeightsAndResidual's
    r->meanWeightedRes = s[CH_SUMRESW] / n;                // SE3Tracker.cpp:789
    r->meanUnweightedRes = s[CH_SUMRESU] / s[CH_GOOD];     // :1028
    r->warpedSize = (int)n;
    r->pointUsage = s[CH_USAGE] / s[CH_REFNUM];            // :1018
    r->goodCount = s[CH_GOOD];
    r->badCount = s[CH_BAD];
    r->meanRes = s[CH_SIGNED] / s[CH_GOOD];                // :1021
    const float sxx = s[CH_SXX], syy = s[CH_SYY], sx = s[CH_SX], sy = s[CH_SY], sw = s[CH_SW];
    r->affine_a_lastIt = sqrtf((syy - sy * sy / sw) / (sxx - sx * sx / sw));   // :1023-1024
    r->affine_b_lastIt = (sy - r->affine_a_lastIt * sx) / sw;
    r->sxx = sxx; r->syy = syy; r->sx = sx; r->sy = sy; r->sw = sw;
}
