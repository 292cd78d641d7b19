// oracle/ref_driver.cpp -- TEST INFRASTRUCTURE (checker only; never linked or loaded by the product).
//
// C entry points over the REFERENCE'S OWN classes, compiled from the unmodified sources under
// /root/reference/lsd_slam_core/src (recipe: oracle/ref_build.py -> oracle/_ref/liblsd_ref*.so):
//   lsd_slam::Frame            DataStructures/Frame.{h,cpp}, FrameMemory.cpp, FramePoseStruct.cpp
//   lsd_slam::TrackingReference Tracking/TrackingReference.{h,cpp}
//   lsd_slam::SE3Tracker       Tracking/SE3Tracker.{h,cpp}, LGSX.h
//   lsd_slam::DepthMap         DepthEstimation/DepthMap.{h,cpp}, DepthMapPixelHypothesis.{h,cpp}
//   lsd_slam::Sim3Tracker      Tracking/Sim3Tracker.{h,cpp}
//   lsd_slam::UndistorterPTAM  util/Undistorter.{h,cpp} (and Undistorter::getUndistorterForFile's dispatch)
//   Sophus                     thirdparty/Sophus/sophus/{so3,se3,rxso3,sim3}.hpp (vendored, unmodified)
// against the stand-in headers of oracle/ref_shim/ (Eigen 3.2 subset, Boost.Thread -> std, OpenCV debug images).
// The exported names and structs are those of oracle/lsd_oracle.h, so oracle/pyoracle.py drives this library and the
// hand-written C restatement (oracle/lsd_oracle.c) through the same binding and tests/test_ref_pin.py compares the two.
//
// This file contains no algorithm: it constructs the reference's objects, calls their methods and copies fields out.
// Private members are reached with the `#define private public` test idiom in THIS translation unit only (the
// reference's own .cpp files are compiled untouched; access specifiers do not change the Itanium-ABI layout).
#include <algorithm>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <deque>
#include <functional>
#include <iostream>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <sstream>
#include <string>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>
#include <chrono>
#include <limits>
#include <stdexcept>
#include <new>
#include <sys/time.h>
#include <unistd.h>

#include "Eigen/Core"                       // shim (no private members of its own that matter)
#include "boost/thread.hpp"
#include "opencv2/core/core.hpp"

#define private public
#define protected public
#include "util/settings.h"
#include "util/SophusUtil.h"
#include "DataStructures/Frame.h"
#include "DataStructures/FramePoseStruct.h"
#include "DepthEstimation/DepthMapPixelHypothesis.h"
#include "DepthEstimation/DepthMap.h"
#include "Tracking/TrackingReference.h"
#include "Tracking/SE3Tracker.h"
#include "Tracking/Sim3Tracker.h"
#include "IOWrapper/ImageDisplay.h"
#include "util/Undistorter.h"
#undef private
#undef protected

#include "lsd_oracle.h"

using namespace lsd_slam;

// ---- headless IOWrapper (the reference selects an implementation per platform: IOWrapper/OpenCV, IOWrapper/Android) ----
namespace lsd_slam { namespace Util {
void displayImage(const char*, const cv::Mat&, bool) {}
int waitKey(int) { return -1; }
int waitKeyNoConsume(int) { return -1; }
void closeAllWindows() {}
} }

static_assert(sizeof(DepthMapPixelHypothesis) == sizeof(lsdo_hyp), "hypothesis record must be 32 bytes");
static_assert(sizeof(bool) == 1, "refPixelWasGood is exported as bytes");

struct lsdo_frame {
    std::shared_ptr<Frame> f;
    int w, h;
    std::vector<float> grad_scratch[PYRAMID_LEVELS];
};
struct lsdo_depthmap {
    DepthMap* d;
    Eigen::Matrix3f K;
    int w, h;
    // keyframes stay alive as long as the DepthMap may hold their activeMutex (DepthMap.h:111-112), whatever order the
    // caller drops its handles in
    std::vector<std::shared_ptr<Frame> > keep;
};

static lsdo_globals G_shadow;

// The reference's buffer pool (FrameMemory.cpp:67-95) hands recycled, uncleared buffers to buildMaxGradients, which reads
// two never-written rows of them (Frame.cpp:721-734; SURVEY.md App. A-12): the reference is not deterministic there.
// With the switch on (default in the scalar / parity build) the pool is emptied before every call that can build such a
// buffer, so that each one is a fresh zero-filled allocation -- the definition the oracle and the CUDA path use.  The
// timing build leaves the pool alone (recycling is part of what the reference's speed is).
#if defined(ENABLE_SSE)
static int g_deterministic_pool = 0;
#else
static int g_deterministic_pool = 1;
#endif
static inline void flushPool() { if (g_deterministic_pool) FrameMemory::getInstance().releaseBuffes(); }

static Eigen::Matrix3f toK(const float K[9])
{
    Eigen::Matrix3f m;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) m(i, j) = K[i * 3 + j];
    return m;
}
static void qtFromSE3(const SE3& T, double qt[7])
{
    const Eigen::Quaterniond& q = T.unit_quaternion();
    qt[0] = q.x(); qt[1] = q.y(); qt[2] = q.z(); qt[3] = q.w();
    qt[4] = T.translation()[0]; qt[5] = T.translation()[1]; qt[6] = T.translation()[2];
}
static SE3 se3FromQt(const double qt[7])
{
    // SE3Group(const Quaternion&, const Point&) normalises the quaternion (so3.hpp: SO3Group(quat) -> normalize())
    return SE3(Eigen::Quaterniond(qt[3], qt[0], qt[1], qt[2]), Eigen::Vector3d(qt[4], qt[5], qt[6]));
}
static Sophus::SE3f se3fFromQt(const float qt[7])
{
    return Sophus::SE3f(Eigen::Quaternionf(qt[3], qt[0], qt[1], qt[2]), Eigen::Vector3f(qt[4], qt[5], qt[6]));
}
static Sim3 sim3FromQts(const double q[8])
{
    Sim3 s(Sophus::RxSO3d(q[7], Sophus::SO3d(Eigen::Quaterniond(q[3], q[0], q[1], q[2]))), Eigen::Vector3d(q[4], q[5], q[6]));
    return s;
}
static void qtsFromSim3(const Sim3& s, double q[8])
{
    const double sc = s.scale();
    Eigen::Quaterniond u = s.quaternion();
    u.normalize();
    q[0] = u.x(); q[1] = u.y(); q[2] = u.z(); q[3] = u.w();
    q[4] = s.translation()[0]; q[5] = s.translation()[1]; q[6] = s.translation()[2];
    q[7] = sc;
}
static void applyTrackSettings(DenseDepthTrackerSettings& d, const lsdo_track_settings* s)
{
    if (!s) return;
    d.lambdaSuccessFac = s->lambdaSuccessFac;
    d.lambdaFailFac = s->lambdaFailFac;
    for (int i = 0; i < PYRAMID_LEVELS; i++) {
        d.lambdaInitial[i] = s->lambdaInitial[i];
        d.stepSizeMin[i] = s->stepSizeMin[i];
        d.convergenceEps[i] = s->convergenceEps[i];
        d.maxItsPerLvl[i] = s->maxItsPerLvl[i];
    }
    d.huber_d = s->huber_d;
    d.var_weight = s->var_weight;
}

extern "C" {

void lsdo_ref_deterministic_pool(int on) { g_deterministic_pool = on; }

const char* lsdo_flavour(void)
{
#if defined(ENABLE_SSE)
    return "reference-compiled (lsd_slam_core sources, ENABLE_SSE)";
#else
    return "reference-compiled (lsd_slam_core sources, scalar)";
#endif
}

void lsdo_default_globals(lsdo_globals* g)
{
    g->minUseGrad = 5; g->cameraPixelNoise2 = 16; g->depthSmoothingFactor = 1;
    g->allowNegativeIdepths = 1; g->useSubpixelStereo = 1; g->useAffineLightningEstimation = 1;
    g->multiThreading = 1;
#if defined(ENABLE_SSE)
    g->useSSE = 1;
#else
    g->useSSE = 0;
#endif
    g->exactAffineSums = 0;
    g->exactTrackingSums = 0;          // diagnostic switches of the C restatement: no equivalent in the reference
}
void lsdo_set_globals(const lsdo_globals* g)
{
    G_shadow = *g;
    minUseGrad = g->minUseGrad; cameraPixelNoise2 = g->cameraPixelNoise2; depthSmoothingFactor = g->depthSmoothingFactor;
    allowNegativeIdepths = g->allowNegativeIdepths != 0; useSubpixelStereo = g->useSubpixelStereo != 0;
    useAffineLightningEstimation = g->useAffineLightningEstimation != 0; multiThreading = g->multiThreading != 0;
    // useSSE is a compile-time property of this library (ENABLE_SSE); exactAffineSums does not exist in the reference
}
void lsdo_get_globals(lsdo_globals* g)
{
    lsdo_default_globals(g);
    g->minUseGrad = minUseGrad; g->cameraPixelNoise2 = cameraPixelNoise2; g->depthSmoothingFactor = depthSmoothingFactor;
    g->allowNegativeIdepths = allowNegativeIdepths; g->useSubpixelStereo = useSubpixelStereo;
    g->useAffineLightningEstimation = useAffineLightningEstimation; g->multiThreading = multiThreading;
}
void lsdo_default_track_settings(lsdo_track_settings* s)
{
    DenseDepthTrackerSettings d;                           // util/settings.h:355-402
    s->lambdaSuccessFac = d.lambdaSuccessFac; s->lambdaFailFac = d.lambdaFailFac;
    for (int i = 0; i < PYRAMID_LEVELS; i++) {
        s->lambdaInitial[i] = d.lambdaInitial[i]; s->stepSizeMin[i] = d.stepSizeMin[i];
        s->convergenceEps[i] = d.convergenceEps[i]; s->maxItsPerLvl[i] = d.maxItsPerLvl[i];
    }
    s->huber_d = d.huber_d; s->var_weight = d.var_weight;
}

// ---- Sophus (vendored) ----
void lsdo_se3d_exp(const double a[6], double qt[7])
{
    Eigen::Matrix<double, 6, 1> v; for (int i = 0; i < 6; i++) v[i] = a[i];
    qtFromSE3(SE3::exp(v), qt);
}
void lsdo_se3d_mul(const double a[7], const double b[7], double out[7]) { qtFromSE3(se3FromQt(a) * se3FromQt(b), out); }
void lsdo_se3d_inverse(const double a[7], double out[7]) { qtFromSE3(se3FromQt(a).inverse(), out); }
void lsdo_se3d_log(const double a[7], double out[6])
{
    Eigen::Matrix<double, 6, 1> v = se3FromQt(a).log();
    for (int i = 0; i < 6; i++) out[i] = v[i];
}
void lsdo_se3d_matrix(const double a[7], double R[9], double t[3])
{
    SE3 T = se3FromQt(a);
    Eigen::Matrix3d m = T.rotationMatrix();
    for (int i = 0; i < 3; i++) { for (int j = 0; j < 3; j++) R[i * 3 + j] = m(i, j); t[i] = T.translation()[i]; }
}
void lsdo_se3f_exp(const float a[6], float qt[7])
{
    Eigen::Matrix<float, 6, 1> v; for (int i = 0; i < 6; i++) v[i] = a[i];
    Sophus::SE3f T = Sophus::SE3f::exp(v);
    const Eigen::Quaternionf& q = T.unit_quaternion();
    qt[0] = q.x(); qt[1] = q.y(); qt[2] = q.z(); qt[3] = q.w();
    for (int i = 0; i < 3; i++) qt[4 + i] = T.translation()[i];
}
static void qtFromSE3f(const Sophus::SE3f& T, float qt[7])
{
    const Eigen::Quaternionf& q = T.unit_quaternion();
    qt[0] = q.x(); qt[1] = q.y(); qt[2] = q.z(); qt[3] = q.w();
    for (int i = 0; i < 3; i++) qt[4 + i] = T.translation()[i];
}
// raw (not re-normalised) construction so that products and inverses see exactly the coefficients passed in
static Sophus::SE3f se3fRaw(const float qt[7])
{
    Sophus::SE3f T;
    std::memcpy(T.data(), qt, 7 * sizeof(float));      // SE3Group::data(): quaternion (x,y,z,w) then translation (se3.hpp)
    return T;
}
void lsdo_se3f_mul(const float a[7], const float b[7], float out[7]) { qtFromSE3f(se3fRaw(a) * se3fRaw(b), out); }
void lsdo_se3f_inverse(const float a[7], float out[7]) { qtFromSE3f(se3fRaw(a).inverse(), out); }
void lsdo_se3f_matrix(const float a[7], float R[9], float t[3])
{
    Sophus::SE3f T = se3fRaw(a);
    Eigen::Matrix3f m = T.rotationMatrix();
    for (int i = 0; i < 3; i++) { for (int j = 0; j < 3; j++) R[i * 3 + j] = m(i, j); t[i] = T.translation()[i]; }
}
void lsdo_sim3d_exp(const double a[7], double out[8])
{
    Eigen::Matrix<double, 7, 1> v; for (int i = 0; i < 7; i++) v[i] = a[i];
    qtsFromSim3(Sim3::exp(v), out);
}
void lsdo_sim3d_mul(const double a[8], const double b[8], double out[8]) { qtsFromSim3(sim3FromQts(a) * sim3FromQts(b), out); }
void lsdo_sim3d_inverse(const double a[8], double out[8]) { qtsFromSim3(sim3FromQts(a).inverse(), out); }
int lsdo_ldlt6_solve(const float A[36], const float b[6], float x[6])
{
    Matrix6x6 M; Vector6 v;
    for (int i = 0; i < 6; i++) { for (int j = 0; j < 6; j++) M(i, j) = A[i * 6 + j]; v[i] = b[i]; }
    Vector6 r = M.ldlt().solve(v);
    for (int i = 0; i < 6; i++) x[i] = r[i];
    return 0;
}
void lsdo_mat3_inverse(const float K[9], float Kinv[9])
{
    Eigen::Matrix3f m = toK(K).inverse();
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Kinv[i * 3 + j] = m(i, j);
}

// ---- Frame ----
lsdo_frame* lsdo_frame_create_u8(int id, int w, int h, const float K[9], const uint8_t* image)
{
    flushPool();
    lsdo_frame* o = new lsdo_frame;
    o->w = w; o->h = h;
    o->f.reset(new Frame(id, w, h, toK(K), 0.0, image));
    return o;
}
void lsdo_frame_destroy(lsdo_frame* f) { delete f; }
int lsdo_frame_id(const lsdo_frame* f) { return f->f->id(); }
int lsdo_frame_width(const lsdo_frame* f, int l) { return f->f->width(l); }
int lsdo_frame_height(const lsdo_frame* f, int l) { return f->f->height(l); }
const float* lsdo_frame_image(lsdo_frame* f, int l) { return f->f->image(l); }
const float* lsdo_frame_gradients(lsdo_frame* f, int l)
{
    // the reference leaves rows 0 / h-1 and the 4th component undefined (Frame.cpp:643-680, recycled pool buffers);
    // the oracle defines them as zero (SURVEY App. A-7, A-12).  Copy the defined cells, zero the rest.
    const int w = f->f->width(l), h = f->f->height(l);
    const Eigen::Vector4f* g = f->f->gradients(l);
    std::vector<float>& s = f->grad_scratch[l];
    s.assign((size_t)w * h * 4, 0.0f);
    for (int y = 1; y < h - 1; y++)
        for (int x = 0; x < w; x++) {
            const Eigen::Vector4f& v = g[x + y * w];
            float* d = &s[(size_t)(x + y * w) * 4];
            d[0] = v[0]; d[1] = v[1]; d[2] = v[2];
        }
    return s.data();
}
const float* lsdo_frame_maxGradients(lsdo_frame* f, int l) { flushPool(); return f->f->maxGradients(l); }
const float* lsdo_frame_idepth(lsdo_frame* f, int l) { return f->f->idepth(l); }
const float* lsdo_frame_idepthVar(lsdo_frame* f, int l) { return f->f->idepthVar(l); }
void lsdo_frame_K(const lsdo_frame* f, int l, float K[9], float Kinv[9])
{
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) { K[i * 3 + j] = f->f->K(l)(i, j); Kinv[i * 3 + j] = f->f->KInv(l)(i, j); }
}
uint8_t* lsdo_frame_refPixelWasGood(lsdo_frame* f) { return reinterpret_cast<uint8_t*>(f->f->refPixelWasGood()); }
uint8_t* lsdo_frame_refPixelWasGoodNoCreate(lsdo_frame* f) { return reinterpret_cast<uint8_t*>(f->f->refPixelWasGoodNoCreate()); }
void lsdo_frame_clear_refPixelWasGood(lsdo_frame* f) { f->f->clear_refPixelWasGood(); }
void lsdo_frame_setDepthFromGroundTruth(lsdo_frame* f, const float* depth, float cov_scale) { flushPool(); f->f->setDepthFromGroundTruth(depth, cov_scale); }
void lsdo_frame_setDepth(lsdo_frame* f, const lsdo_hyp* d) { f->f->setDepth(reinterpret_cast<const DepthMapPixelHypothesis*>(d)); }
int lsdo_frame_numMappablePixels(lsdo_frame* f) { flushPool(); f->f->maxGradients(0); return f->f->numMappablePixels; }
float lsdo_frame_meanIdepth(const lsdo_frame* f) { return f->f->meanIdepth; }
int lsdo_frame_numPoints(const lsdo_frame* f) { return f->f->numPoints; }
int lsdo_frame_depthHasBeenUpdatedFlag(const lsdo_frame* f) { return f->f->depthHasBeenUpdatedFlag; }
void lsdo_frame_set_depthHasBeenUpdatedFlag(lsdo_frame* f, int v) { f->f->depthHasBeenUpdatedFlag = v != 0; }
float lsdo_frame_initialTrackedResidual(const lsdo_frame* f) { return f->f->initialTrackedResidual; }
void lsdo_frame_set_initialTrackedResidual(lsdo_frame* f, float v) { f->f->initialTrackedResidual = v; }
void lsdo_frame_get_thisToParent(const lsdo_frame* f, double qts[8]) { qtsFromSim3(f->f->pose->thisToParent_raw, qts); }
void lsdo_frame_set_thisToParent(lsdo_frame* f, const double qts[8], lsdo_frame* parent)
{
    f->f->pose->thisToParent_raw = sim3FromQts(qts);
    f->f->pose->trackingParent = parent ? parent->f->pose : nullptr;
    f->f->pose->invalidateCache();
}
int lsdo_frame_numFramesTrackedOnThis(const lsdo_frame* f) { return f->f->numFramesTrackedOnThis; }
int lsdo_frame_numMappedOnThis(const lsdo_frame* f) { return f->f->numMappedOnThis; }
void lsdo_frame_set_counters(lsdo_frame* f, int tracked, int mapped) { f->f->numFramesTrackedOnThis = tracked; f->f->numMappedOnThis = mapped; }
void lsdo_frame_takeReActivationData(lsdo_frame* f, const lsdo_hyp* dm)
{
    f->f->takeReActivationData(const_cast<DepthMapPixelHypothesis*>(reinterpret_cast<const DepthMapPixelHypothesis*>(dm)));
}
const float* lsdo_frame_idepth_reAct(const lsdo_frame* f) { return f->f->idepth_reAct(); }
const float* lsdo_frame_idepthVar_reAct(const lsdo_frame* f) { return f->f->idepthVar_reAct(); }
const uint8_t* lsdo_frame_validity_reAct(const lsdo_frame* f) { return f->f->validity_reAct(); }

// ---- TrackingReference ----
int lsdo_make_point_cloud(lsdo_frame* kf, int level, float* posData, float* gradData, float* colorAndVarData, int* pointPosInXYGrid)
{
    TrackingReference ref;
    ref.importFrame(kf->f.get());
    ref.makePointCloud(level);
    const int n = ref.numData[level];
    for (int i = 0; i < n; i++) {
        if (posData) for (int k = 0; k < 3; k++) posData[i * 3 + k] = ref.posData[level][i][k];
        if (gradData) for (int k = 0; k < 2; k++) gradData[i * 2 + k] = ref.gradData[level][i][k];
        if (colorAndVarData) for (int k = 0; k < 2; k++) colorAndVarData[i * 2 + k] = ref.colorAndVarData[level][i][k];
        if (pointPosInXYGrid) pointPosInXYGrid[i] = ref.pointPosInXYGrid[level][i];
    }
    ref.invalidate();
    return n;
}

// ---- SE3Tracker ----
int lsdo_se3_eval(lsdo_frame* kf, lsdo_frame* frame, int level, const float refToFrame_qt[7], float affine_a, float affine_b,
                  const lsdo_track_settings* s, int writeGoodMask, lsdo_eval_result* out)
{
    std::memset(out, 0, sizeof(*out));
    SE3Tracker t(kf->w, kf->h, kf->f->K(0));
    applyTrackSettings(t.settings, s);
    TrackingReference ref;
    ref.importFrame(kf->f.get());
    ref.makePointCloud(level);
    t.affineEstimation_a = affine_a; t.affineEstimation_b = affine_b;
    Sophus::SE3f T = se3fFromQt(refToFrame_qt);
    int* idx = writeGoodMask ? ref.pointPosInXYGrid[level] : nullptr;
#if defined(ENABLE_SSE)
    out->meanUnweightedRes = t.calcResidualAndBuffersSSE(ref.posData[level], ref.colorAndVarData[level], idx, ref.numData[level], frame->f.get(), T, level, false);
    out->meanWeightedRes = t.calcWeightsAndResidualSSE(T);
    LGS6 ls;
    t.calculateWarpUpdateSSE(ls);
#else
    out->meanUnweightedRes = t.calcResidualAndBuffers(ref.posData[level], ref.colorAndVarData[level], idx, ref.numData[level], frame->f.get(), T, level, false);
    out->meanWeightedRes = t.calcWeightsAndResidual(T);
    LGS6 ls;
    t.calculateWarpUpdate(ls);
#endif
    for (int i = 0; i < 6; i++) { for (int j = 0; j < 6; j++) out->A[i * 6 + j] = ls.A(i, j); out->b[i] = ls.b[i]; }
    out->lsError = ls.error;
    out->warpedSize = t.buf_warped_size;
    out->pointUsage = t.pointUsage; out->goodCount = t.lastGoodCount; out->badCount = t.lastBadCount; out->meanRes = t.lastMeanRes;
    out->affine_a_lastIt = t.affineEstimation_a_lastIt; out->affine_b_lastIt = t.affineEstimation_b_lastIt;
    out->sxx = out->syy = out->sx = out->sy = out->sw = std::numeric_limits<float>::quiet_NaN();   // locals in the reference
    ref.invalidate();
    return 0;
}

int lsdo_se3_track(lsdo_frame* kf, lsdo_frame* frame, const double frameToRef_init_qt[7], const lsdo_track_settings* s, lsdo_track_result* out)
{
    std::memset(out, 0, sizeof(*out));
    SE3Tracker t(kf->w, kf->h, kf->f->K(0));
    applyTrackSettings(t.settings, s);
    TrackingReference ref;
    ref.importFrame(kf->f.get());
    const int tracked0 = kf->f->numFramesTrackedOnThis;
    SE3 res = t.trackFrame(&ref, frame->f.get(), se3FromQt(frameToRef_init_qt));
    (void)tracked0;
    qtFromSE3(res, out->frameToRef_qt);
    out->pointUsage = t.pointUsage; out->lastGoodCount = t.lastGoodCount; out->lastBadCount = t.lastBadCount;
    out->lastMeanRes = t.lastMeanRes; out->lastResidual = t.lastResidual;
    out->affineEstimation_a = t.affineEstimation_a; out->affineEstimation_b = t.affineEstimation_b;
    out->diverged = t.diverged; out->trackingWasGood = t.trackingWasGood;
    for (int i = 0; i < PYRAMID_LEVELS; i++) out->numCalcResidualCalls[i] = out->numCalcWarpUpdateCalls[i] = -1;  // locals in the reference (SE3Tracker.cpp:310-311)
    out->initialTrackedResidual = frame->f->initialTrackedResidual;
    ref.invalidate();
    return 0;
}

// ---- Sim3Tracker (Tracking/Sim3Tracker.cpp:149-382) ----
// one evaluation as trackFrameSim3 runs it per LM step: calcSim3Buffers -> calcSim3WeightsAndResidual -> calcSim3LGS
int lsdo_sim3_eval(lsdo_frame* ref_kf, lsdo_frame* frame, int level, const double refToFrame_qts[8], float affine_a, float affine_b,
                   const lsdo_track_settings* s, lsdo_sim3_eval_result* out)
{
    std::memset(out, 0, sizeof(*out));
    Sim3Tracker t(ref_kf->w, ref_kf->h, ref_kf->f->K(0));
    applyTrackSettings(t.settings, s);
    TrackingReference ref;
    ref.importFrame(ref_kf->f.get());
    ref.makePointCloud(level);
    t.affineEstimation_a = affine_a; t.affineEstimation_b = affine_b;
    const Sim3 T = sim3FromQts(refToFrame_qts);
    LGS7 ls7;
#if defined(ENABLE_SSE)
    t.calcSim3BuffersSSE(&ref, frame->f.get(), T, level, false);
    Sim3ResidualStruct r = t.calcSim3WeightsAndResidualSSE(T);
    t.calcSim3LGSSSE(ls7);
#else
    t.calcSim3Buffers(&ref, frame->f.get(), T, level, false);
    Sim3ResidualStruct r = t.calcSim3WeightsAndResidual(T);
    t.calcSim3LGS(ls7);
#endif
    for (int i = 0; i < 7; i++) { for (int j = 0; j < 7; j++) out->A[i * 7 + j] = ls7.A(i, j); out->b[i] = ls7.b[i]; }
    out->num_constraints = (int)ls7.num_constraints;
    out->sumResD = r.sumResD; out->sumResP = r.sumResP; out->numTermsD = r.numTermsD; out->numTermsP = r.numTermsP;
    out->mean = r.mean; out->meanD = r.meanD; out->meanP = r.meanP;
    out->warpedSize = t.buf_warped_size; out->pointUsage = t.pointUsage;
    out->affine_a_lastIt = t.affineEstimation_a_lastIt; out->affine_b_lastIt = t.affineEstimation_b_lastIt;
    ref.invalidate();
    return 0;
}

int lsdo_sim3_track(lsdo_frame* ref_kf, lsdo_frame* frame, const double frameToRef_init_qts[8], int startLevel, int finalLevel,
                    const lsdo_track_settings* s, lsdo_sim3_result* out)
{
    std::memset(out, 0, sizeof(*out));
    Sim3Tracker t(ref_kf->w, ref_kf->h, ref_kf->f->K(0));
    applyTrackSettings(t.settings, s);
    TrackingReference ref;
    ref.importFrame(ref_kf->f.get());
    Sim3 res = t.trackFrameSim3(&ref, frame->f.get(), sim3FromQts(frameToRef_init_qts), startLevel, finalLevel);
    qtsFromSim3(res, out->frameToRef_qts);
    for (int i = 0; i < 7; i++) for (int j = 0; j < 7; j++) out->lastSim3Hessian[i * 7 + j] = t.lastSim3Hessian(i, j);
    out->lastResidual = t.lastResidual; out->lastDepthResidual = t.lastDepthResidual; out->lastPhotometricResidual = t.lastPhotometricResidual;
    out->pointUsage = t.pointUsage; out->affineEstimation_a = t.affineEstimation_a; out->affineEstimation_b = t.affineEstimation_b;
    out->diverged = t.diverged;
    for (int i = 0; i < PYRAMID_LEVELS; i++) out->numCalcResidualCalls[i] = out->numCalcWarpUpdateCalls[i] = -1;   // locals in the reference
    ref.invalidate();
    return 0;
}

// ---- permaRef (Frame.cpp:149-174, SE3Tracker.cpp:121-272) ----
int lsdo_frame_setPermaRef(lsdo_frame* kf, float* posData, float* colorAndVarData)
{
    TrackingReference ref;
    ref.importFrame(kf->f.get());
    kf->f->setPermaRef(&ref);
    const int n = kf->f->permaRefNumPts;
    for (int i = 0; i < n; i++) {
        if (posData) for (int k = 0; k < 3; k++) posData[i * 3 + k] = kf->f->permaRef_posData[i][k];
        if (colorAndVarData) for (int k = 0; k < 2; k++) colorAndVarData[i * 2 + k] = kf->f->permaRef_colorAndVarData[i][k];
    }
    ref.invalidate();
    return n;
}
float lsdo_ref_checkPermaRefOverlap(lsdo_frame* kf, const double refToFrame_qt[7])
{
    SE3Tracker t(kf->w, kf->h, kf->f->K(0));
    return t.checkPermaRefOverlap(kf->f.get(), se3FromQt(refToFrame_qt));
}
int lsdo_ref_trackFrameOnPermaref(lsdo_frame* kf, lsdo_frame* frame, const double refToFrame_qt[7], lsdo_track_result* out)
{
    std::memset(out, 0, sizeof(*out));
    SE3Tracker t(kf->w, kf->h, kf->f->K(0));
    SE3 res = t.trackFrameOnPermaref(kf->f.get(), frame->f.get(), se3FromQt(refToFrame_qt));
    qtFromSE3(res, out->frameToRef_qt);             // referenceToFrame, as the C restatement returns it
    out->pointUsage = t.pointUsage; out->lastGoodCount = t.lastGoodCount; out->lastBadCount = t.lastBadCount;
    out->lastMeanRes = t.lastMeanRes; out->lastResidual = t.lastResidual;
    out->affineEstimation_a = t.affineEstimation_a; out->affineEstimation_b = t.affineEstimation_b;
    out->diverged = t.diverged; out->trackingWasGood = t.trackingWasGood;
    for (int i = 0; i < PYRAMID_LEVELS; i++) out->numCalcResidualCalls[i] = out->numCalcWarpUpdateCalls[i] = -1;   // not counted there
    return 0;
}

// ---- DepthMap ----
lsdo_depthmap* lsdo_depthmap_create(int w, int h, const float K[9])
{
    lsdo_depthmap* o = new lsdo_depthmap;
    o->K = toK(K); o->w = w; o->h = h;
    o->d = new DepthMap(w, h, o->K);
    return o;
}
void lsdo_depthmap_destroy(lsdo_depthmap* d) { delete d->d; d->keep.clear(); delete d; }
void lsdo_depthmap_reset(lsdo_depthmap* d) { d->d->reset(); }
void lsdo_depthmap_initializeFromGTDepth(lsdo_depthmap* d, lsdo_frame* f) { flushPool(); d->keep.push_back(f->f); d->d->initializeFromGTDepth(f->f.get()); }
void lsdo_depthmap_initializeRandomly(lsdo_depthmap* d, lsdo_frame* f) { flushPool(); d->keep.push_back(f->f); d->d->initializeRandomly(f->f.get()); }
void lsdo_depthmap_updateKeyframe(lsdo_depthmap* d, lsdo_frame** refs, int n)
{
    std::deque<std::shared_ptr<Frame> > q;
    for (int i = 0; i < n; i++) q.push_back(refs[i]->f);
    d->d->updateKeyframe(q);
}
void lsdo_depthmap_createKeyFrame(lsdo_depthmap* d, lsdo_frame* nk) { flushPool(); d->keep.push_back(nk->f); d->d->createKeyFrame(nk->f.get()); while (d->keep.size() > 3) d->keep.erase(d->keep.begin()); }
void lsdo_depthmap_finalizeKeyFrame(lsdo_depthmap* d) { d->d->finalizeKeyFrame(); }
const lsdo_hyp* lsdo_depthmap_current(const lsdo_depthmap* d) { return reinterpret_cast<const lsdo_hyp*>(d->d->currentDepthMap); }
void lsdo_depthmap_set_current(lsdo_depthmap* d, const lsdo_hyp* h) { std::memcpy(d->d->currentDepthMap, h, sizeof(lsdo_hyp) * d->w * d->h); }
const int* lsdo_depthmap_integral(const lsdo_depthmap* d) { return d->d->validityIntegralBuffer; }
// individual passes (private members of the reference class, called as they are)
void lsdo_depthmap_observeDepth(lsdo_depthmap* dd, lsdo_frame** refs, int n)
{
    DepthMap* d = dd->d;
    // the set-up block of updateKeyframe (DepthMap.cpp:1079-1107) for frames tracked on the active keyframe
    d->oldest_referenceFrame = refs[0]->f.get();
    d->newest_referenceFrame = refs[n - 1]->f.get();
    d->referenceFrameByID.clear();
    d->referenceFrameByID_offset = d->oldest_referenceFrame->id();
    for (int i = 0; i < n; i++) {
        Frame* frame = refs[i]->f.get();
        Sim3 refToKf;
        if (frame->pose->trackingParent->frameID == d->activeKeyFrame->id()) refToKf = frame->pose->thisToParent_raw;
        else refToKf = d->activeKeyFrame->getScaledCamToWorld().inverse() * frame->getScaledCamToWorld();
        frame->prepareForStereoWith(d->activeKeyFrame, refToKf, d->K, 0);
        while ((int)d->referenceFrameByID.size() + d->referenceFrameByID_offset <= frame->id()) d->referenceFrameByID.push_back(frame);
    }
    d->resetCounters();
    d->observeDepth();
}
void lsdo_depthmap_regularizeFillHoles(lsdo_depthmap* d) { d->d->regularizeDepthMapFillHoles(); }
void lsdo_depthmap_regularize(lsdo_depthmap* d, int removeOcclusions, int validityTH) { d->d->regularizeDepthMap(removeOcclusions != 0, validityTH); }
void lsdo_depthmap_propagateDepth(lsdo_depthmap* d, lsdo_frame* nk) { flushPool(); d->d->propagateDepth(nk->f.get()); }
void lsdo_depthmap_last_timings(const lsdo_depthmap* d, float out_ms[8])
{
    const DepthMap* m = d->d;
    const float v[8] = { m->msUpdate, m->msCreate, m->msFinalize, m->msObserve, m->msRegularize, m->msPropagate, m->msFillHoles, m->msSetDepth };
    std::memcpy(out_ms, v, sizeof(v));
}
// the stereo constants Frame::prepareForStereoWith leaves in the reference frame (Frame.cpp:295-317), for direct comparison
void lsdo_ref_prepareForStereoWith(lsdo_frame* frame, lsdo_frame* kf, const double thisToOther_qts[8], const float K[9], float out[30])
{
    frame->f->prepareForStereoWith(kf->f.get(), sim3FromQts(thisToOther_qts), toK(K), 0);
    Frame* f = frame->f.get();
    int k = 0;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) out[k++] = f->K_otherToThis_R(i, j);
    for (int i = 0; i < 3; i++) out[k++] = f->K_otherToThis_t[i];
    for (int i = 0; i < 3; i++) out[k++] = f->otherToThis_t[i];
    for (int i = 0; i < 3; i++) out[k++] = f->thisToOther_t[i];
    for (int i = 0; i < 3; i++) out[k++] = f->otherToThis_R_row0[i];
    for (int i = 0; i < 3; i++) out[k++] = f->otherToThis_R_row1[i];
    for (int i = 0; i < 3; i++) out[k++] = f->otherToThis_R_row2[i];
    out[k++] = f->distSquared;
    out[k++] = (float)f->referenceID;
    out[k++] = (float)f->referenceLevel;
}

// ---- UndistorterPTAM (util/Undistorter.cpp:38-411) ----
// The reference constructs the class from a calibration file only.  The object lives in zero-filled storage: for "none" the
// constructor leaves outputCalibration unset (Undistorter.cpp:140-143) and reads it at :270-273, and zero is what the library's
// adapter uses there (lsd_host.cpp), so this makes that case defined and the same on both sides.
struct lsdo_ref_undistorter {
    alignas(UndistorterPTAM) unsigned char storage[sizeof(UndistorterPTAM)];
    UndistorterPTAM* u;
};

lsdo_ref_undistorter* lsdo_ref_undistorter_open(const char* path)
{
    lsdo_ref_undistorter* o = new lsdo_ref_undistorter;
    std::memset(o->storage, 0, sizeof(o->storage));
    o->u = new (o->storage) UndistorterPTAM(path);
    return o;
}
void lsdo_ref_undistorter_close(lsdo_ref_undistorter* o)
{
    o->u->~UndistorterPTAM();
    delete o;
}
// info = valid, in_w, in_h, out_w, out_h; K as main_on_images.cpp:164-167 reads getK() (float of (0,0), (1,1), (2,0), (2,1))
void lsdo_ref_undistorter_info(const lsdo_ref_undistorter* o, int info[5], float K[9])
{
    const UndistorterPTAM* u = o->u;
    info[0] = u->isValid() ? 1 : 0;
    info[1] = u->getInputWidth(); info[2] = u->getInputHeight();
    info[3] = u->getOutputWidth(); info[4] = u->getOutputHeight();
    std::memset(K, 0, 9 * sizeof(float));
    K[0] = (float)u->getK().at<double>(0, 0);
    K[4] = (float)u->getK().at<double>(1, 1);
    K[2] = (float)u->getK().at<double>(2, 0);
    K[5] = (float)u->getK().at<double>(2, 1);
    K[8] = 1;
}
// remapX / remapY (out_w * out_h floats each); 0 when the reference built none (an invalid file)
int lsdo_ref_undistorter_tables(const lsdo_ref_undistorter* o, float* remapX, float* remapY)
{
    const UndistorterPTAM* u = o->u;
    if (!u->remapX || !u->remapY) return 0;
    const size_t n = (size_t)u->out_width * u->out_height;
    std::memcpy(remapX, u->remapX, n * sizeof(float));
    std::memcpy(remapY, u->remapY, n * sizeof(float));
    return 1;
}
// undistort() of an in_h x in_w image into out (capacity `cap` bytes); returns rows * 65536 + cols of the result, which is the
// input itself when the reference passes it through (Undistorter.cpp:357-375)
int lsdo_ref_undistorter_undistort(const lsdo_ref_undistorter* o, const uint8_t* image, int in_w, int in_h, uint8_t* out, int cap)
{
    cv::Mat img(in_h, in_w, CV_8U, const_cast<uint8_t*>(image));
    cv::Mat res;
    o->u->undistort(img, res);
    if ((long long)res.rows * res.cols > cap) return -1;
    std::memcpy(out, res.data, (size_t)res.rows * res.cols);
    return res.rows * 65536 + res.cols;
}
// Undistorter::getUndistorterForFile (:38-88): 0 for its null result, 1 for an UndistorterPTAM.  A file whose first line holds
// 8 numbers constructs UndistorterOpenCV, whose OpenCV calls this library does not have: callers must not pass one.
int lsdo_ref_undistorter_for_file(const char* path)
{
    Undistorter* u = Undistorter::getUndistorterForFile(path);
    if (!u) return 0;
    const int kind = dynamic_cast<UndistorterPTAM*>(u) ? 1 : 2;
    delete u;
    return kind;
}

// The C oracle's parsed-line API (oracle/lsd_oracle_undistort.inc) over the reference's class: the four lines are written to a
// temporary file with %.9g, which sscanf("%f") reads back to the same floats, and the file goes through the constructor above.
int lsdo_undistorter_ptam_prepare(const float inputCalibration[5], int in_width, int in_height, const float outputCalibrationIn[5],
                                  int out_width, int out_height, float* remapX, float* remapY, float K_out[9])
{
    if (in_width <= 0 || in_height <= 0 || out_width <= 0 || out_height <= 0) return -1;
    const char* tmpdir = std::getenv("TMPDIR");
    const std::string tpl = std::string(tmpdir && *tmpdir ? tmpdir : "/tmp") + "/lsdo_undistorter_XXXXXX";
    std::vector<char> name(tpl.begin(), tpl.end());
    name.push_back(0);
    const int fd = mkstemp(name.data());
    if (fd < 0) return -1;
    FILE* f = fdopen(fd, "w");
    const float* ic = inputCalibration;
    const float* oc = outputCalibrationIn;
    std::fprintf(f, "%.9g %.9g %.9g %.9g %.9g\n%d %d\n", ic[0], ic[1], ic[2], ic[3], ic[4], in_width, in_height);
    if (oc[0] == -1) std::fprintf(f, "crop\n");
    else if (oc[0] == -2) std::fprintf(f, "full\n");
    else std::fprintf(f, "%.9g %.9g %.9g %.9g %.9g\n", oc[0], oc[1], oc[2], oc[3], oc[4]);
    std::fprintf(f, "%d %d\n", out_width, out_height);
    std::fclose(f);
    lsdo_ref_undistorter* o = lsdo_ref_undistorter_open(name.data());
    unlink(name.data());
    int info[5];
    float K[9];
    lsdo_ref_undistorter_info(o, info, K);
    int status = -1;
    if (info[0]) {
        if (K_out) std::memcpy(K_out, K, sizeof(K));
        if (remapX && remapY) lsdo_ref_undistorter_tables(o, remapX, remapY);
        status = (in_height == out_height && in_width == out_width && ic[4] == 0) ? 1 : 0;
    }
    lsdo_ref_undistorter_close(o);
    return status;
}

// UndistorterPTAM::undistort (:380-410) with the caller's tables.  The object is built from no file (not valid, no tables) and
// then given the tables and sizes; undistort() addresses the input through in_width alone (:402) and compares the image's rows
// with in_height only to refuse a wrong size, so in_height is set to the rows of the wrapper it is handed.  The distortion is
// set non-zero so that the pass-through of :370-375 is not taken (callers handle that case themselves, as pyoracle does).
void lsdo_undistort(const float* remapX, const float* remapY, int in_width, int out_width, int out_height,
                    const uint8_t* image, uint8_t* data)
{
    lsdo_ref_undistorter* o = lsdo_ref_undistorter_open("");
    UndistorterPTAM* u = o->u;
    const int rows = 1;
    u->valid = true;
    u->in_width = in_width; u->in_height = rows;
    u->out_width = out_width; u->out_height = out_height;
    u->inputCalibration[4] = 1;
    u->remapX = const_cast<float*>(remapX);
    u->remapY = const_cast<float*>(remapY);
    cv::Mat img(rows, in_width, CV_8U, const_cast<uint8_t*>(image));
    cv::Mat res;
    u->undistort(img, res);
    std::memcpy(data, res.data, (size_t)out_width * out_height);
    u->remapX = u->remapY = nullptr;              // the caller's arrays: not the reference's to free
    lsdo_ref_undistorter_close(o);
}

}  // extern "C"
