// lsd_host.cpp -- implementation of lsd_host.h over the C ABI.  See the header for the reference citations.
#include "lsd_host.h"

#include <algorithm>
#include <cstdio>
#include <fstream>
#include <iterator>
#include <string>

#include <cmath>
#include <cstdlib>
#include <cstring>

namespace lsd_slam {

// util/settings.cpp:80-88
float minUseGrad = 5;
float cameraPixelNoise2 = 4 * 4;
float depthSmoothingFactor = 1;
bool allowNegativeIdepths = true;
bool useSubpixelStereo = true;
bool useAffineLightningEstimation = true;

static void qmul(const double a[4], const double b[4], double o[4])
{
    double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    double y = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    double z = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
    o[0] = x; o[1] = y; o[2] = z; o[3] = w;
}
static void qrot(const double q[4], const double v[3], double o[3])
{
    double ux = q[1] * v[2] - q[2] * v[1], uy = q[2] * v[0] - q[0] * v[2], uz = q[0] * v[1] - q[1] * v[0];
    ux += ux; uy += uy; uz += uz;
    o[0] = v[0] + q[3] * ux + (q[1] * uz - q[2] * uy);
    o[1] = v[1] + q[3] * uy + (q[2] * ux - q[0] * uz);
    o[2] = v[2] + q[3] * uz + (q[0] * uy - q[1] * ux);
}
static void qnorm(double q[4])
{
    double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for (int i = 0; i < 4; i++) q[i] /= n;
}
SE3 SE3::inverse() const
{   // thirdparty/Sophus/sophus/se3.hpp:167-172
    SE3 r;
    r.q[0] = -q[0]; r.q[1] = -q[1]; r.q[2] = -q[2]; r.q[3] = q[3];
    qnorm(r.q);
    double nt[3] = { -t[0], -t[1], -t[2] };
    qrot(r.q, nt, r.t);
    return r;
}
SE3 SE3::operator*(const SE3& o) const
{   // se3.hpp:239-259
    SE3 r;
    double rt[3];
    qrot(q, o.t, rt);
    qmul(q, o.q, r.q);
    qnorm(r.q);
    for (int i = 0; i < 3; i++) r.t[i] = t[i] + rt[i];
    return r;
}

Sim3 Sim3::inverse() const
{
    Sim3 r;
    r.q[0] = -q[0]; r.q[1] = -q[1]; r.q[2] = -q[2]; r.q[3] = q[3];
    qnorm(r.q);
    r.s = 1.0 / s;
    double nt[3] = { -t[0], -t[1], -t[2] }, rt[3];
    qrot(r.q, nt, rt);
    for (int i = 0; i < 3; i++) r.t[i] = r.s * rt[i];
    return r;
}
Sim3 Sim3::operator*(const Sim3& o) const
{
    Sim3 r;
    double rt[3];
    qrot(q, o.t, rt);
    qmul(q, o.q, r.q);
    qnorm(r.q);
    r.s = s * o.s;
    for (int i = 0; i < 3; i++) r.t[i] = t[i] + s * rt[i];
    return r;
}
Sim3 FramePoseStruct::getCamToWorld(int recursionDepth) const
{
    if (recursionDepth >= 5000) throw LsdGpuError("FramePoseStruct::getCamToWorld: assert(recursionDepth < 5000)");
    if (trackingParent == nullptr) return Sim3();
    return trackingParent->getCamToWorld(recursionDepth + 1) * thisToParent_raw;
}

DeviceContext::DeviceContext(int device, int w, int h, const Matrix3f& K, int maxFrames) : w_(w), h_(h), maxFrames_(maxFrames)
{
    memory_.reset(new FrameMemory(*this, 10 + 20));       // maxLoopClosureCandidates + 20, settings.cpp:97 / FrameMemory.cpp:153
    int rc = lsdgpu_create(device, w, h, K.m, maxFrames, &ctx_);
    if (rc != 0) {
        std::string msg = ctx_ ? lsdgpu_last_error(ctx_) : "lsdgpu_create failed (bad size: width and height must be multiples of 16)";
        if (ctx_) lsdgpu_destroy(ctx_);
        ctx_ = nullptr;
        throw LsdGpuError(msg);
    }
    followGlobals();                                      // a context starts with the values in force, not the defaults
}
DeviceContext::~DeviceContext() { if (ctx_) lsdgpu_destroy(ctx_); }
void DeviceContext::check(int rc, const char* where) const
{
    if (rc != 0) throw LsdGpuError(std::string(where) + ": " + lsdgpu_last_error(ctx_));
}
void DeviceContext::setInputFormat(int format) { check(lsdgpu_set_input_format(ctx_, format), "DeviceContext::setInputFormat"); }
void DeviceContext::followGlobals()
{
    lsdgpu_globals want, have;
    want.minUseGrad = minUseGrad;
    want.cameraPixelNoise2 = cameraPixelNoise2;
    want.depthSmoothingFactor = depthSmoothingFactor;
    want.allowNegativeIdepths = allowNegativeIdepths;
    want.useSubpixelStereo = useSubpixelStereo;
    want.useAffineLightningEstimation = useAffineLightningEstimation;
    check(lsdgpu_get_globals(ctx_, &have), "DeviceContext::followGlobals");
    if (std::memcmp(&want, &have, sizeof(want)) != 0)     // six 4-byte fields, no padding
        check(lsdgpu_set_globals(ctx_, &want), "DeviceContext::followGlobals");
}

FrameMemory::FrameMemory(DeviceContext& dev, int maxActive) : dev_(dev), maxActive_(maxActive) {}

void FrameMemory::minimizeLeastRecent()
{
    const int activeKf = lsdgpu_depth_active_keyframe(dev_.raw());
    for (auto it = activeFrames.rbegin(); it != activeFrames.rend(); ++it) {
        Frame* f = *it;
        if (f->id() == activeKf || std::find(held_.begin(), held_.end(), f) != held_.end()) continue;
        activeFrames.erase(std::next(it).base());
        minimize(f);
        return;
    }
    throw LsdGpuError("FrameMemory: no frame slot can be freed: every active frame is the active keyframe or in use by this call "
                      "(raise max_frames)");
}
void FrameMemory::minimize(Frame* frame)
{
    frame->minimizeOnDevice();
    frame->isActive = false;
    deviceRecords_.push_front(frame);
}
void FrameMemory::makeRoom()
{
    std::lock_guard<std::recursive_mutex> l(mu_);
    while ((int)activeFrames.size() >= dev_.maxFrames()) minimizeLeastRecent();
}
void FrameMemory::activateFrame(Frame* frame)
{
    dev_.followGlobals();
    std::lock_guard<std::recursive_mutex> l(mu_);
    if (frame->isActive) {
        activeFrames.remove(frame);
    } else {
        makeRoom();
        dev_.check(lsdgpu_frame_activate(dev_.raw(), frame->id()), "FrameMemory::activateFrame");     // from either tier
        frame->isActive = true;
        deviceRecords_.remove(frame);
    }
    activeFrames.push_front(frame);
}
void FrameMemory::deactivateFrame(Frame* frame)
{
    dev_.followGlobals();
    std::lock_guard<std::recursive_mutex> l(mu_);
    if (!frame->isActive) return;
    activeFrames.remove(frame);
    minimize(frame);
}
void FrameMemory::pruneActiveFrames()
{
    dev_.followGlobals();
    std::lock_guard<std::recursive_mutex> l(mu_);
    while ((int)activeFrames.size() > maxActive_) minimizeLeastRecent();
    while (maxDeviceRecords_ >= 0 && (int)deviceRecords_.size() > maxDeviceRecords_) {
        Frame* f = deviceRecords_.back();
        dev_.check(lsdgpu_frame_offload(dev_.raw(), f->id()), "FrameMemory::pruneActiveFrames");
        deviceRecords_.pop_back();
    }
}

ActiveFrames::ActiveFrames(FrameMemory& memory, std::initializer_list<Frame*> frames)
    : ActiveFrames(memory, std::vector<Frame*>(frames)) {}
ActiveFrames::ActiveFrames(FrameMemory& memory, const std::vector<Frame*>& frames) : memory_(memory)
{
    std::lock_guard<std::recursive_mutex> l(memory_.mu_);
    try {
        for (Frame* f : frames) {
            memory_.activateFrame(f);
            memory_.held_.push_back(f);
            n_++;
        }
    } catch (...) {
        memory_.held_.resize(memory_.held_.size() - n_);
        throw;
    }
}
ActiveFrames::~ActiveFrames()
{
    std::lock_guard<std::recursive_mutex> l(memory_.mu_);
    memory_.held_.resize(memory_.held_.size() - n_);
}

Frame::Frame(DeviceContext& dev, int id, int width, int height, const Matrix3f&, double timestamp, const unsigned char* image, bool distorted)
    : dev_(dev), id_(id), w_(width), h_(height), timestamp_(timestamp)
{
    dev_.followGlobals();
    pose = new FramePoseStruct();
    pose->frameID = id;
    FrameMemory& m = dev_.frameMemory();
    std::lock_guard<std::recursive_mutex> l(m.mu_);
    m.makeRoom();
    dev_.check(distorted ? lsdgpu_frame_upload_distorted_u8(dev_.raw(), id, image) : lsdgpu_frame_upload_u8(dev_.raw(), id, image), "Frame::Frame");
    m.activeFrames.push_front(this);                    // Frame.cpp:35-54 leaves a new frame active
}
Frame::~Frame()
{
    {
        FrameMemory& m = dev_.frameMemory();
        std::lock_guard<std::recursive_mutex> l(m.mu_);
        if (isActive) m.activeFrames.remove(this);
        else m.deviceRecords_.remove(this);
    }
    lsdgpu_frame_release(dev_.raw(), id_);      // may fail for the active keyframe: DepthMap::invalidate() first
    delete pose;
}
void Frame::minimizeOnDevice() { dev_.check(lsdgpu_frame_minimize(dev_.raw(), id_), "Frame::minimizeInMemory"); }
bool Frame::minimizeInMemory()
{
    dev_.frameMemory().deactivateFrame(this);
    return true;
}
void Frame::getActiveLock() { dev_.frameMemory().activateFrame(this); }
void Frame::setDepthFromGroundTruth(const float* depth, float cov_scale)
{
    dev_.followGlobals();
    getActiveLock();                                                    // Frame.cpp:247
    dev_.check(lsdgpu_frame_set_depth_gt(dev_.raw(), id_, depth, cov_scale), "Frame::setDepthFromGroundTruth");
}
void Frame::clear_refPixelWasGood()
{
    if (!isActive) return;                                              // minimizeInMemory cleared it, Frame.cpp:388
    dev_.followGlobals();
    dev_.check(lsdgpu_frame_clear_good_mask(dev_.raw(), id_), "Frame::clear_refPixelWasGood");
}
float Frame::meanIdepth()
{
    dev_.followGlobals();
    float m = 1; int n = 0, f = 0;
    dev_.check(lsdgpu_frame_get_depth_stats(dev_.raw(), id_, &m, &n, &f), "Frame::meanIdepth");
    return m;
}
int Frame::numPoints()
{
    dev_.followGlobals();
    float m = 1; int n = 0, f = 0;
    dev_.check(lsdgpu_frame_get_depth_stats(dev_.raw(), id_, &m, &n, &f), "Frame::numPoints");
    return n;
}
bool Frame::depthHasBeenUpdatedFlag() const
{
    dev_.followGlobals();
    int f = 0;
    dev_.check(lsdgpu_frame_get_depth_stats(dev_.raw(), id_, nullptr, nullptr, &f), "Frame::depthHasBeenUpdatedFlag");
    return f != 0;
}
void Frame::downloadIdepth(int level, std::vector<float>& idepth, std::vector<float>& idepthVar)
{
    dev_.followGlobals();
    if (level > 0) getActiveLock();                                     // levels 1..4 are rebuilt on activation (Frame::require)
    size_t n = (size_t)width(level) * height(level);
    idepth.resize(n); idepthVar.resize(n);
    dev_.check(lsdgpu_frame_download(dev_.raw(), id_, LSDGPU_BUF_IDEPTH, level, idepth.data()), "Frame::idepth");
    dev_.check(lsdgpu_frame_download(dev_.raw(), id_, LSDGPU_BUF_IDEPTH_VAR, level, idepthVar.data()), "Frame::idepthVar");
}
void Frame::setPermaRef(TrackingReference* reference)
{   // Frame.cpp:149-174
    if (reference->frameID != id_)                                      // assert(reference->frameID == id()), :151
        throw LsdGpuError("Frame::setPermaRef: the TrackingReference holds frame " + std::to_string(reference->frameID) + ", not frame " +
                          std::to_string(id_));
    dev_.followGlobals();
    ActiveFrames held(dev_.frameMemory(), { this });                    // the TrackingReference holds the keyframe's active lock
    int n = 0;
    dev_.check(lsdgpu_frame_set_perma_ref(dev_.raw(), id_, &n), "Frame::setPermaRef");
    permaRefNumPts = n;
}
void Frame::downloadRefPixelWasGood(std::vector<unsigned char>& mask)
{
    dev_.followGlobals();
    getActiveLock();
    mask.resize((size_t)width(1) * height(1));
    dev_.check(lsdgpu_frame_download(dev_.raw(), id_, LSDGPU_BUF_GOODMASK, 1, mask.data()), "Frame::refPixelWasGood");
}

void TrackingReference::importFrame(Frame* sourceKF)
{
    sourceKF->dev().followGlobals();
    sourceKF->getActiveLock();                                          // TrackingReference.cpp:74
    keyframe = sourceKF;
    frameID = sourceKF->id();
    sourceKF->dev().check(lsdgpu_ref_import(sourceKF->dev().raw(), frameID), "TrackingReference::importFrame");
}

SE3Tracker::SE3Tracker(DeviceContext& dev, int w, int h, const Matrix3f&) : dev_(dev), width_(w), height_(h)
{
    if (w != dev.width() || h != dev.height()) throw LsdGpuError("SE3Tracker: size differs from the device context");
}

static void se3ToQt(const SE3& a, double o[7])
{
    for (int i = 0; i < 4; i++) o[i] = a.q[i];
    for (int i = 0; i < 3; i++) o[4 + i] = a.t[i];
}

SE3 SE3Tracker::trackFrame(TrackingReference* reference, Frame* frame, const SE3& frameToReference_initialEstimate)
{
    dev_.followGlobals();
    double init[7];
    se3ToQt(frameToReference_initialEstimate, init);
    ActiveFrames held(dev_.frameMemory(), { reference->keyframe, frame });   // SE3Tracker.cpp:286; the keyframe's levels live in its slot
    lsdgpu_track_result r;
    dev_.check(lsdgpu_se3_track(dev_.raw(), reference->keyframe->id(), frame->id(), init, &settings, mode, &r), "SE3Tracker::trackFrame");
    pointUsage = r.pointUsage; lastGoodCount = r.lastGoodCount; lastBadCount = r.lastBadCount;
    lastMeanRes = r.lastMeanRes; lastResidual = r.lastResidual;
    affineEstimation_a = r.affineEstimation_a; affineEstimation_b = r.affineEstimation_b;
    diverged = r.diverged != 0; trackingWasGood = r.trackingWasGood != 0;
    SE3 out;
    if (diverged) return out;                                         // SE3(), SE3Tracker.cpp:324-329
    for (int i = 0; i < 4; i++) out.q[i] = r.frameToRef_qt[i];
    for (int i = 0; i < 3; i++) out.t[i] = r.frameToRef_qt[4 + i];
    if (trackingWasGood) reference->keyframe->numFramesTrackedOnThis++;   // :479-480
    frame->initialTrackedResidual = r.initialTrackedResidual;         // :482
    frame->pose->thisToParent_raw = sim3FromSE3(out, 1);              // :483
    frame->pose->trackingParent = reference->keyframe->pose;          // :484
    return out;
}

float SE3Tracker::checkPermaRefOverlap(Frame* reference, SE3 referenceToFrame)
{   // reads only the permaRef, which a minimized keyframe keeps in its record
    dev_.followGlobals();
    const int kfId = reference->id();
    double qt[7];
    se3ToQt(referenceToFrame, qt);
    float usage = 0;
    if (int rc = lsdgpu_perma_overlap_batch(dev_.raw(), 1, &kfId, qt, &usage))
        dev_.check(rc, ("SE3Tracker::checkPermaRefOverlap (keyframe " + std::to_string(kfId) + ")").c_str());
    pointUsage = usage;                                               // :155
    return pointUsage;
}

SE3 SE3Tracker::trackFrameOnPermaref(Frame* reference, Frame* frame, SE3 referenceToFrame)
{
    dev_.followGlobals();
    ActiveFrames held(dev_.frameMemory(), { frame });                 // :170; the reference's permaRef needs no slot
    const int kfId = reference->id();
    double init[7];
    se3ToQt(referenceToFrame, init);
    lsdgpu_track_result r;
    if (int rc = lsdgpu_perma_track_batch(dev_.raw(), 1, &kfId, frame->id(), init, &r))
        dev_.check(rc, ("SE3Tracker::trackFrameOnPermaref (keyframe " + std::to_string(kfId) + ")").c_str());
    // the last calcResidualAndBuffers sets these, also on the diverging one
    pointUsage = r.pointUsage; lastGoodCount = r.lastGoodCount; lastBadCount = r.lastBadCount; lastMeanRes = r.lastMeanRes;
    affineEstimation_a = r.affineEstimation_a; affineEstimation_b = r.affineEstimation_b;
    diverged = r.diverged != 0; trackingWasGood = r.trackingWasGood != 0;
    SE3 out;
    if (diverged) return out;                                         // SE3(), :180-185, :215-220; lastResidual keeps its value
    lastResidual = r.lastResidual;                                    // :265
    for (int i = 0; i < 4; i++) out.q[i] = r.frameToRef_qt[i];        // referenceToFrame, :271
    for (int i = 0; i < 3; i++) out.t[i] = r.frameToRef_qt[4 + i];
    return out;
}

Sim3Tracker::Sim3Tracker(DeviceContext& dev, int w, int h, const Matrix3f&) : dev_(dev), width_(w), height_(h)
{
    if (w != dev.width() || h != dev.height()) throw LsdGpuError("Sim3Tracker: size differs from the device context");
    lastSim3Hessian.setZero();
}

static void sim3ToQts(const Sim3& a, double o[8])
{
    for (int i = 0; i < 4; i++) o[i] = a.q[i];
    for (int i = 0; i < 3; i++) o[4 + i] = a.t[i];
    o[7] = a.s;
}

Sim3 Sim3Tracker::take(const lsdgpu_sim3_result& r)
{
    // members a diverged / rejected tracking leaves untouched keep their previous values (Sim3Tracker.cpp:184-187, 212-217)
    pointUsage = r.pointUsage;
    affineEstimation_a = r.affineEstimation_a; affineEstimation_b = r.affineEstimation_b;
    diverged = r.diverged != 0;
    Sim3 out;                                                          // Sim3()
    bool hessianZero = true;
    for (float v : r.lastSim3Hessian) hessianZero = hessianZero && v == 0.f;
    if (diverged && hessianZero) return out;                           // :184-187, :231-235
    for (int i = 0; i < 49; i++) lastSim3Hessian.m[i] = r.lastSim3Hessian[i];     // :360 (also zeroed by :215)
    if (diverged || hessianZero) return out;                           // :363-367, :212-217
    lastResidual = r.lastResidual; lastDepthResidual = r.lastDepthResidual; lastPhotometricResidual = r.lastPhotometricResidual;
    for (int i = 0; i < 4; i++) out.q[i] = r.frameToRef_qts[i];
    for (int i = 0; i < 3; i++) out.t[i] = r.frameToRef_qts[4 + i];
    out.s = r.frameToRef_qts[7];
    return out;
}

Sim3 Sim3Tracker::trackFrameSim3(TrackingReference* reference, Frame* frame, const Sim3& frameToReference_initialEstimate,
                                 int startLevel, int finalLevel)
{
    dev_.followGlobals();
    double init[8];
    sim3ToQts(frameToReference_initialEstimate, init);
    ActiveFrames held(dev_.frameMemory(), { reference->keyframe, frame });   // Sim3Tracker.cpp:155
    lsdgpu_sim3_result r;
    dev_.check(lsdgpu_sim3_track(dev_.raw(), reference->keyframe->id(), frame->id(), init, startLevel, finalLevel, &settings, &r),
               "Sim3Tracker::trackFrameSim3");
    return take(r);
}

void Sim3Tracker::trackFrameSim3Batch(const std::vector<TrackingReference*>& references, const std::vector<Frame*>& frames,
                                      const std::vector<Sim3>& inits, int startLevel, int finalLevel,
                                      std::vector<Sim3>& frameToReference, std::vector<lsdgpu_sim3_result>& results)
{
    dev_.followGlobals();
    const size_t n = references.size();
    if (frames.size() != n || inits.size() != n) throw LsdGpuError("Sim3Tracker::trackFrameSim3Batch: list lengths differ");
    std::vector<int> refIds(n), frIds(n);
    std::vector<double> q(8 * n);
    std::vector<Frame*> used;
    for (size_t i = 0; i < n; i++) { used.push_back(references[i]->keyframe); used.push_back(frames[i]); }
    ActiveFrames held(dev_.frameMemory(), used);
    for (size_t i = 0; i < n; i++) {
        refIds[i] = references[i]->keyframe->id(); frIds[i] = frames[i]->id();
        sim3ToQts(inits[i], &q[8 * i]);
    }
    results.resize(n);
    dev_.check(lsdgpu_sim3_track_batch(dev_.raw(), (int)n, refIds.data(), frIds.data(), q.data(), startLevel, finalLevel, &settings, results.data()),
               "Sim3Tracker::trackFrameSim3Batch");
    frameToReference.resize(n);
    for (size_t i = 0; i < n; i++) frameToReference[i] = take(results[i]);
}

UndistorterPTAM::UndistorterPTAM(const char* configFileName)
{   // parsing as Undistorter.cpp:100-166; everything after that is lsdgpu_undistorter_ptam_prepare (:171-317)
    for (int i = 0; i < 9; i++) K_.m[i] = 0.f;
    std::ifstream infile(configFileName);
    if (!infile.good()) return;
    std::string l1, l2, l3, l4;
    std::getline(infile, l1); std::getline(infile, l2); std::getline(infile, l3); std::getline(infile, l4);
    float probe[8];
    if (std::sscanf(l1.c_str(), "%f %f %f %f %f %f %f %f", &probe[0], &probe[1], &probe[2], &probe[3], &probe[4], &probe[5], &probe[6], &probe[7]) == 8)
        return;                                                        // OpenCV camera model (:70-79)
    valid = std::sscanf(l1.c_str(), "%f %f %f %f %f", &inputCalibration[0], &inputCalibration[1], &inputCalibration[2],
                        &inputCalibration[3], &inputCalibration[4]) == 5
            && std::sscanf(l2.c_str(), "%d %d", &in_width, &in_height) == 2;
    for (float& v : outputCalibration) v = 0.f;
    bool none = false;
    if (l3 == "crop") outputCalibration[0] = -1;
    else if (l3 == "full") outputCalibration[0] = -2;
    else if (l3 == "none") none = true;                                // "NO RECTIFICATION" (:138-141): explicit zeros
    else if (std::sscanf(l3.c_str(), "%f %f %f %f %f", &outputCalibration[0], &outputCalibration[1], &outputCalibration[2],
                         &outputCalibration[3], &outputCalibration[4]) != 5)
        valid = false;
    (void)none;
    if (std::sscanf(l4.c_str(), "%d %d", &out_width, &out_height) != 2) valid = false;
    if (!valid) return;
    remapX.resize((size_t)out_width * out_height);
    remapY.resize((size_t)out_width * out_height);
    const int st = lsdgpu_undistorter_ptam_prepare(inputCalibration, in_width, in_height, outputCalibration, out_width, out_height,
                                                   remapX.data(), remapY.data(), K_.m);
    if (st < 0) { valid = false; return; }
    passThrough = (st == 1);
}

void UndistorterPTAM::install(DeviceContext& dev) const
{
    dev.followGlobals();
    if (!valid) throw LsdGpuError("UndistorterPTAM: invalid calibration");
    if (dev.width() != out_width || dev.height() != out_height) throw LsdGpuError("UndistorterPTAM: output size differs from the device context");
    dev.check(lsdgpu_set_undistorter(dev.raw(), in_width, in_height, passThrough ? nullptr : remapX.data(), passThrough ? nullptr : remapY.data()),
              "UndistorterPTAM::install");
}

void UndistorterPTAM::undistort(DeviceContext& dev, const unsigned char* image, unsigned char* result) const
{
    dev.followGlobals();
    dev.check(lsdgpu_undistort_u8(dev.raw(), image, result), "UndistorterPTAM::undistort");
}

UndistorterOpenCV::UndistorterOpenCV(const char* configFileName)
{   // parsing as Undistorter.cpp:449-513; the tables are lsdgpu_undistorter_opencv_prepare (:515-558)
    for (int i = 0; i < 9; i++) K_.m[i] = 0.f;
    for (float& v : inputCalibration) v = 0.f;
    std::ifstream infile(configFileName);
    if (!infile.good()) return;
    std::string l1, l2, l3, l4;
    std::getline(infile, l1); std::getline(infile, l2); std::getline(infile, l3); std::getline(infile, l4);
    float* ic = inputCalibration;
    valid = std::sscanf(l1.c_str(), "%f %f %f %f %f %f %f %f", &ic[0], &ic[1], &ic[2], &ic[3], &ic[4], &ic[5], &ic[6], &ic[7]) == 8
            && std::sscanf(l2.c_str(), "%d %d", &in_width, &in_height) == 2;
    int mode = 0;                                                      // "none" / anything else: not rectifying (:493-502)
    if (l3 == "crop") mode = -1;
    else if (l3 == "full") mode = -2;
    if (std::sscanf(l4.c_str(), "%d %d", &out_width, &out_height) != 2) valid = false;
    if (!valid || mode == 0 || out_width <= 0 || out_height <= 0) { valid = false; return; }
    map1_.resize((size_t)2 * out_width * out_height);
    map2_.resize((size_t)out_width * out_height);
    double K_new[9];
    valid = lsdgpu_undistorter_opencv_prepare(ic, in_width, in_height, mode, out_width, out_height, map1_.data(), map2_.data(),
                                              K_new, K_.m) == 0;
}

void UndistorterOpenCV::install(DeviceContext& dev) const
{
    dev.followGlobals();
    if (!valid) throw LsdGpuError("UndistorterOpenCV: invalid calibration");
    if (dev.width() != out_width || dev.height() != out_height) throw LsdGpuError("UndistorterOpenCV: output size differs from the device context");
    dev.check(lsdgpu_set_undistorter_opencv(dev.raw(), in_width, in_height, map1_.data(), map2_.data()), "UndistorterOpenCV::install");
}

void UndistorterOpenCV::undistort(DeviceContext& dev, const unsigned char* image, unsigned char* result) const
{
    dev.followGlobals();
    dev.check(lsdgpu_undistort_u8(dev.raw(), image, result), "UndistorterOpenCV::undistort");
}

Undistorter* getUndistorterForFile(const char* configFilename)
{   // Undistorter.cpp:38-88 (the search for the file in the working directory and the prints left out)
    std::ifstream f(configFilename);
    if (!f.good()) return nullptr;
    std::string l1;
    std::getline(f, l1);
    f.close();
    float ic[8];
    Undistorter* u;
    if (std::sscanf(l1.c_str(), "%f %f %f %f %f %f %f %f", &ic[0], &ic[1], &ic[2], &ic[3], &ic[4], &ic[5], &ic[6], &ic[7]) == 8)
        u = new UndistorterOpenCV(configFilename);
    else
        u = new UndistorterPTAM(configFilename);
    if (!u->isValid()) { delete u; return nullptr; }
    return u;
}

DepthMap::DepthMap(DeviceContext& dev, int w, int h, const Matrix3f&) : dev_(dev), width_(w), height_(h)
{
    if (w != dev.width() || h != dev.height()) throw LsdGpuError("DepthMap: size differs from the device context");
    reset();
}
void DepthMap::reset()
{
    dev_.followGlobals();
    dev_.check(lsdgpu_depth_reset(dev_.raw()), "DepthMap::reset");
}
void DepthMap::invalidate()
{
    dev_.followGlobals();
    activeKeyFrame = nullptr;
    dev_.check(lsdgpu_depth_invalidate(dev_.raw()), "DepthMap::invalidate");
}
void DepthMap::initializeFromGTDepth(Frame* new_frame)
{
    dev_.followGlobals();
    new_frame->getActiveLock();                                         // DepthMap.cpp:969
    dev_.check(lsdgpu_depth_init_from_gt(dev_.raw(), new_frame->id()), "DepthMap::initializeFromGTDepth");
    activeKeyFrame = new_frame;
}
void DepthMap::initializeRandomly(Frame* new_frame)
{   // DepthMap.cpp:883-916 on the device, drawing from the process's rand() stream and leaving it where the reference's loop would
    dev_.followGlobals();
    new_frame->getActiveLock();                                         // DepthMap.cpp:885
    // initstate() switches rand() to `tmp` and returns the word before the live table: 5 * rear + type (glibc's MAX_TYPES == 5),
    // then the table; setstate() of the same pointer switches back and reads that word again
    int32_t tmp[32];
    int32_t* live = (int32_t*)initstate(1, (char*)tmp, sizeof(tmp));
    if (!live) throw LsdGpuError("DepthMap::initializeRandomly: cannot read the rand() state");
    lsdgpu_rand_state st;
    std::memset(&st, 0, sizeof(st));
    st.type = live[0] % 5;
    st.rear = st.type == 0 ? 0 : live[0] / 5;
    static const int kDeg[5] = { 1, 7, 15, 31, 63 };                    // table words per type (stdlib/random_r.c)
    const int deg = st.type >= 0 && st.type < 5 ? kDeg[st.type] : 0;
    std::memcpy(st.r, live + 1, (size_t)deg * 4);
    const int rc = lsdgpu_depth_init_random(dev_.raw(), new_frame->id(), &st, nullptr);
    if (rc == 0) {
        live[0] = st.type == 0 ? 0 : 5 * st.rear + st.type;
        std::memcpy(live + 1, st.r, (size_t)deg * 4);
    }
    setstate((char*)live);
    dev_.check(rc, "DepthMap::initializeRandomly");
    activeKeyFrame = new_frame;
}
void DepthMap::setFromExistingKF(Frame* kf)
{   // DepthMap.cpp:920-962
    dev_.followGlobals();
    kf->getActiveLock();                                                // :924; rebuilds the levels of a minimized keyframe
    dev_.check(lsdgpu_depth_set_from_existing_kf(dev_.raw(), kf->id()), "DepthMap::setFromExistingKF");
    kf->numMappedOnThis = 0; kf->numFramesTrackedOnThis = 0;            // :932-933
    activeKeyFrame = kf;
}
void DepthMap::setFromExistingKF(Frame* kf, const float* idepth, const float* idepthVar, const unsigned char* validity)
{   // DepthMap.cpp:920-962
    dev_.followGlobals();
    kf->getActiveLock();                                                // DepthMap.cpp:924
    std::vector<lsdgpu_hyp> hyp((size_t)width_ * height_);
    std::memset(hyp.data(), 0, hyp.size() * sizeof(lsdgpu_hyp));
    for (size_t i = 0; i < hyp.size(); i++) {
        lsdgpu_hyp& h = hyp[i];
        if (idepthVar[i] > 0) {
            h.isValid = 1; h.blacklisted = 0; h.nextStereoFrameMinID = 0; h.validity_counter = validity[i];
            h.idepth = idepth[i]; h.idepth_var = idepthVar[i]; h.idepth_smoothed = -1; h.idepth_var_smoothed = -1;
        } else {
            h.isValid = 0;
            h.blacklisted = (idepthVar[i] == -2) ? -2 : 0;
        }
    }
    kf->numMappedOnThis = 0; kf->numFramesTrackedOnThis = 0;
    dev_.check(lsdgpu_depth_set_hypotheses(dev_.raw(), kf->id(), hyp.data(), 1, 0), "DepthMap::setFromExistingKF");
    activeKeyFrame = kf;
}
void DepthMap::updateKeyframe(std::deque<std::shared_ptr<Frame>> referenceFrames)
{
    dev_.followGlobals();
    if (!isValid()) throw LsdGpuError("DepthMap::updateKeyframe: assert(isValid())");
    std::vector<Frame*> used{ activeKeyFrame };
    for (auto& f : referenceFrames) used.push_back(f.get());            // the device reads their images and masks
    ActiveFrames held(dev_.frameMemory(), used);
    std::vector<lsdgpu_ref_desc> refs;
    for (auto& f : referenceFrames) {
        if (!f->hasTrackingParent()) throw LsdGpuError("DepthMap::updateKeyframe: assert(frame->hasTrackingParent())");   // :1085
        lsdgpu_ref_desc d;
        std::memset(&d, 0, sizeof(d));
        d.frame_id = f->id();
        d.tracked_on_kf = f->pose->trackingParent->frameID == activeKeyFrame->id();                    // :1096
        if (!d.tracked_on_kf) {
            // :1087-1099: "tracked on a different frame ... While this should work, it is not recommended."
            const Sim3 refToKf = activeKeyFrame->getScaledCamToWorld().inverse() * f->getScaledCamToWorld();
            for (int i = 0; i < 4; i++) d.refToKf_qts[i] = refToKf.q[i];
            for (int i = 0; i < 3; i++) d.refToKf_qts[4 + i] = refToKf.t[i];
            d.refToKf_qts[7] = refToKf.s;
        }
        refs.push_back(d);
    }
    // the device keeps its own copy of the counters the skip-ahead logic reads (DepthMap.cpp:454)
    dev_.check(lsdgpu_frame_set_counters(dev_.raw(), activeKeyFrame->id(), activeKeyFrame->numFramesTrackedOnThis, activeKeyFrame->numMappedOnThis),
               "DepthMap::updateKeyframe");
    dev_.check(lsdgpu_depth_update_keyframe_refs(dev_.raw(), refs.data(), (int)refs.size()), "DepthMap::updateKeyframe");
    activeKeyFrame->numMappedOnThis++;
    activeKeyFrame->numMappedOnThisTotal++;
}
void DepthMap::createKeyFrame(Frame* new_keyframe)
{
    dev_.followGlobals();
    if (!isValid()) throw LsdGpuError("DepthMap::createKeyFrame: assert(isValid())");
    if (!new_keyframe || !new_keyframe->hasTrackingParent()) throw LsdGpuError("DepthMap::createKeyFrame: new keyframe has no tracking parent");
    ActiveFrames held(dev_.frameMemory(), { activeKeyFrame, new_keyframe });   // DepthMap.cpp:1256, :1229
    double qts[8];
    dev_.check(lsdgpu_depth_create_keyframe(dev_.raw(), new_keyframe->id(), qts), "DepthMap::createKeyFrame");
    Sim3 s;
    for (int i = 0; i < 4; i++) s.q[i] = qts[i];
    for (int i = 0; i < 3; i++) s.t[i] = qts[4 + i];
    s.s = qts[7];
    new_keyframe->pose->thisToParent_raw = s;                            // DepthMap.cpp:1305
    activeKeyFrame = new_keyframe;
}
void DepthMap::finalizeKeyFrame()
{
    dev_.followGlobals();
    if (!isValid()) throw LsdGpuError("DepthMap::finalizeKeyFrame: assert(isValid())");
    activeKeyFrame->getActiveLock();
    dev_.check(lsdgpu_depth_finalize_keyframe(dev_.raw()), "DepthMap::finalizeKeyFrame");
}
void DepthMap::download(std::vector<lsdgpu_hyp>& out)
{
    dev_.followGlobals();
    out.resize((size_t)width_ * height_);
    dev_.check(lsdgpu_depth_download(dev_.raw(), out.data()), "DepthMap::download");
}

}  // namespace lsd_slam
