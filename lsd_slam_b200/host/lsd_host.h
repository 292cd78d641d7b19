// lsd_host.h -- C++ host side of the GPU hot path: classes that keep the reference's names, call signatures and
// observable fields for the three seam methods, implemented on top of the C ABI (include/lsdgpu.h).
//
//   lsd_slam::SE3Tracker::trackFrame          Tracking/SE3Tracker.h:65-68
//   lsd_slam::DepthMap::updateKeyframe        DepthEstimation/DepthMap.h:58
//   lsd_slam::DepthMap::createKeyFrame        DepthEstimation/DepthMap.h:63
//
// and the calls SlamSystem's SLAM mode adds (SlamSystem.cpp:405, 496, 1298-1304; TrackableKeyFrameSearch.cpp:126-135;
// Relocalizer.cpp:172-188): Frame::setPermaRef, SE3Tracker::checkPermaRefOverlap / trackFrameOnPermaref and
// DepthMap::setFromExistingKF(Frame*).
//
// The reference's headers need Eigen / Sophus / Boost / OpenCV, none of which exist in this image, so this
// header carries minimal stand-ins (lsd_slam::SE3, Sim3, Matrix3f) with the same semantics; inside
// lsd_slam_core the adapter in INTEGRATION.md maps them 1:1 onto Sophus::SE3d / Sophus::Sim3d / Eigen::Matrix3f.
// Host code only: no CUDA headers, no torch.  Everything device-side sits behind lsdgpu_* calls.
#pragma once

#include <deque>
#include <initializer_list>
#include <list>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/lsdgpu.h"

namespace lsd_slam {

struct Matrix3f {
    float m[9];                                      // row-major
    float operator()(int r, int c) const { return m[r * 3 + c]; }
};

// Sophus::SE3d stand-in: unit quaternion (x,y,z,w) + translation
struct SE3 {
    double q[4] = { 0, 0, 0, 1 };
    double t[3] = { 0, 0, 0 };
    SE3 inverse() const;
    SE3 operator*(const SE3& o) const;
};
// Sophus::Sim3d stand-in
struct Sim3 {
    double q[4] = { 0, 0, 0, 1 };
    double t[3] = { 0, 0, 0 };
    double s = 1.0;
    Sim3 inverse() const;                            // thirdparty/Sophus/sophus/sim3.hpp:169-173
    Sim3 operator*(const Sim3& o) const;             // sim3.hpp:257-260
};
inline Sim3 sim3FromSE3(const SE3& se3, double scale)     // util/SophusUtil.h:53-58
{
    Sim3 r;
    for (int i = 0; i < 4; i++) r.q[i] = se3.q[i];
    for (int i = 0; i < 3; i++) r.t[i] = se3.t[i];
    r.s = scale;
    return r;
}
inline SE3 se3FromSim3(const Sim3& sim3)                  // util/SophusUtil.h:60-63
{
    SE3 r;
    for (int i = 0; i < 4; i++) r.q[i] = sim3.q[i];
    for (int i = 0; i < 3; i++) r.t[i] = sim3.t[i];
    return r;
}

class LsdGpuError : public std::runtime_error {
public:
    explicit LsdGpuError(const std::string& what) : std::runtime_error(what) {}
};

class Frame;
class DeviceContext;
class TrackingReference;

// util/settings.cpp:80-88: the run-time globals the device path reads, with the reference's defaults.  As in the reference they
// are process-wide and read at every use: every adapter call that reaches the device first hands them to its context
// (DeviceContext::followGlobals), so a change takes effect at the next call, on every context driven through the adapter.
// With the adapter these variables are the source of truth: a direct lsdgpu_set_globals on the same context is overwritten
// at the next adapter call.
extern float minUseGrad, cameraPixelNoise2, depthSmoothingFactor;
extern bool allowNegativeIdepths, useSubpixelStereo, useAffineLightningEstimation;

// DataStructures/FrameMemory.h: the active-frame list of FrameMemory (FrameMemory.cpp:129-166), one per DeviceContext.  The
// reference's heap is unbounded; a context has max_frames slots, so activating a frame (or constructing one) with every slot
// taken first minimizes the least recently activated frame that is neither the depth map's active keyframe nor held by a call
// in progress (ActiveFrames).  A call that needs more frames than that leaves free throws LsdGpuError.
// The reference keeps minimized frames in host RAM; here their records stay in device memory unless setMaxDeviceRecords(n) is set:
// pruneActiveFrames then also offloads the least recently minimized records beyond n to host memory (lsdgpu_frame_offload).
class FrameMemory {
public:
    FrameMemory(DeviceContext& dev, int maxActive);
    void activateFrame(Frame* frame);                   // FrameMemory.cpp:129-137 + Frame::require (lsdgpu_frame_activate)
    void deactivateFrame(Frame* frame);                 // FrameMemory.cpp:138-147
    // FrameMemory.cpp:149-166: at most maxActive frames stay active, and at most maxDeviceRecords minimized ones in device memory
    void pruneActiveFrames();
    int maxActiveFrames() const { return maxActive_; }
    void setMaxActiveFrames(int n) { maxActive_ = n; }
    int maxDeviceRecords() const { return maxDeviceRecords_; }
    void setMaxDeviceRecords(int n) { maxDeviceRecords_ = n; }     // < 0: unlimited (the default)

private:
    friend class Frame;
    friend class ActiveFrames;
    void makeRoom();                                    // a free slot for one more active frame
    void minimizeLeastRecent();
    void minimize(Frame* frame);
    DeviceContext& dev_;
    int maxActive_;
    int maxDeviceRecords_ = -1;
    std::list<Frame*> activeFrames;                     // most recently activated first
    std::list<Frame*> deviceRecords_;                   // minimized frames whose record is in device memory, most recent first
    std::vector<Frame*> held_;                          // frames of the calls in progress (ActiveFrames)
    std::recursive_mutex mu_;                           // FrameMemory::activeFramesMutex (tracking and mapping threads)
};

// The frames one device call reads, activated and kept in their slots until the call returns (the shared active locks the
// reference holds for the duration of trackFrame, updateKeyframe, ..., Frame.h:138-141)
class ActiveFrames {
public:
    ActiveFrames(FrameMemory& memory, std::initializer_list<Frame*> frames);
    ActiveFrames(FrameMemory& memory, const std::vector<Frame*>& frames);
    ~ActiveFrames();
    ActiveFrames(const ActiveFrames&) = delete;

private:
    FrameMemory& memory_;
    size_t n_ = 0;
};

// One device context per SlamSystem, shared by every tracker and the depth map of that SlamSystem: the main tracker and the
// DepthMap, the constraint thread's SE3Tracker and Sim3Tracker (SlamSystem.cpp:89-90), TrackableKeyFrameSearch's and the
// Relocalizer's trackers.  Frames live in the context that uploaded them; calls from several threads serialise on the
// context's mutex.
class DeviceContext {
public:
    DeviceContext(int device, int w, int h, const Matrix3f& K, int maxFrames = 16);
    ~DeviceContext();
    DeviceContext(const DeviceContext&) = delete;
    DeviceContext& operator=(const DeviceContext&) = delete;
    lsdgpu_ctx* raw() const { return ctx_; }
    void check(int rc, const char* where) const;
    // the globals above into the context when its values differ (lsdgpu_get_globals / lsdgpu_set_globals); every method of
    // the adapter that reaches the device calls it first (destructors aside: releasing reads no global)
    void followGlobals();
    int width() const { return w_; }
    int height() const { return h_; }
    int maxFrames() const { return maxFrames_; }
    // bound of pruneActiveFrames: maxLoopClosureCandidates + 20 (util/settings.cpp:97)
    FrameMemory& frameMemory() { return *memory_; }
    // the pixel format (LSDGPU_PIX_*) of the installed undistorter's raw images: Frame(.., image, /*distorted=*/true) and
    // Undistorter::undistort then take colour or 4:2:2 camera images and convert them on the device as cv::cvtColor does
    // (LiveSLAMWrapper.cpp:116-121: newImageCallback's cvtColor(img, grayImg, CV_RGB2GRAY) becomes
    // dev.setInputFormat(img.channels() == 1 ? LSDGPU_PIX_MONO8 : img.channels() == 3 ? LSDGPU_PIX_RGB8 : LSDGPU_PIX_RGBA8)).
    // Needs an installed undistorter; lsdgpu_set_input_format.
    void setInputFormat(int format);

private:
    lsdgpu_ctx* ctx_ = nullptr;
    int w_, h_, maxFrames_;
    std::unique_ptr<FrameMemory> memory_;
};

// FramePoseStruct, DataStructures/FramePoseStruct.h (the two members the path touches)
struct FramePoseStruct {
    Sim3 thisToParent_raw;
    FramePoseStruct* trackingParent = nullptr;
    int frameID = -1;
    // FramePoseStruct.cpp:84-105 without the pose-graph members (isOptimized / the cache belong to KeyFrameGraph, out of scope):
    // identity for the first frame, otherwise the parent's absolute pose times thisToParent_raw
    Sim3 getCamToWorld(int recursionDepth = 0) const;
};

// DataStructures/Frame.h -- device-resident frame; host keeps the bookkeeping the callers read
class Frame {
public:
    // `distorted` = true: `image` is the RAW camera image of the installed UndistorterPTAM's input size; undistortion is
    // fused into the pyramid construction on the device (replaces undistort() + this constructor, main_on_images.cpp:238-244)
    Frame(DeviceContext& dev, int id, int width, int height, const Matrix3f& K, double timestamp, const unsigned char* image,
          bool distorted = false);
    ~Frame();
    Frame(const Frame&) = delete;
    int id() const { return id_; }
    int width(int level = 0) const { return w_ >> level; }
    int height(int level = 0) const { return h_ >> level; }
    double timestamp() const { return timestamp_; }
    void setDepthFromGroundTruth(const float* depth, float cov_scale = 1.0f);      // Frame.cpp:245-293
    bool hasTrackingParent() const { return pose->trackingParent != nullptr; }
    Sim3 getScaledCamToWorld() const { return pose->getCamToWorld(); }              // Frame.h:276-280
    void clear_refPixelWasGood();                                                   // Frame.h:439
    float meanIdepth();                                                             // Frame.cpp:234 (lazy D2H)
    int numPoints();
    bool depthHasBeenUpdatedFlag() const;
    // buffers for callers that still need host copies (e.g. Output3DWrapper): explicit downloads
    void downloadIdepth(int level, std::vector<float>& idepth, std::vector<float>& idepthVar);
    void downloadRefPixelWasGood(std::vector<unsigned char>& mask);
    // Frame.cpp:377-395: frees the slot; level 0, the reactivation data and the permaRef stay (lsdgpu_frame_minimize).  Goes
    // through FrameMemory::deactivateFrame so that the next getActiveLock activates the frame again.
    bool minimizeInMemory();
    // Frame.h:138-141: makes the frame active (FrameMemory::activateFrame); the device's calls need the frame in a slot
    void getActiveLock();
    // Frame.cpp:149-174: freezes the keyframe's current level-4 point cloud for the permaRef trackers
    // (lsdgpu_frame_set_perma_ref).  `reference` must hold this frame; otherwise LsdGpuError and nothing changes.
    void setPermaRef(TrackingReference* reference);

    FramePoseStruct* pose;
    bool isActive = true;
    float initialTrackedResidual = 0;
    int numFramesTrackedOnThis = 0, numMappedOnThis = 0, numMappedOnThisTotal = 0;
    int permaRefNumPts = 0;                                                         // Frame.h:176

    DeviceContext& dev() const { return dev_; }

private:
    friend class FrameMemory;
    void minimizeOnDevice();
    DeviceContext& dev_;
    int id_, w_, h_;
    double timestamp_;
};

// Tracking/TrackingReference.h
class TrackingReference {
public:
    Frame* keyframe = nullptr;
    int frameID = -1;
    void importFrame(Frame* sourceKF);                                              // TrackingReference.cpp:71-87
    void invalidate() { keyframe = nullptr; }
};

// util/settings.h:355-402
struct DenseDepthTrackerSettings : lsdgpu_track_settings {
    DenseDepthTrackerSettings() { lsdgpu_default_track_settings(this); }
};

// Tracking/SE3Tracker.h
class SE3Tracker {
public:
    SE3Tracker(DeviceContext& dev, int w, int h, const Matrix3f& K);
    SE3Tracker(const SE3Tracker&) = delete;

    SE3 trackFrame(TrackingReference* reference, Frame* frame, const SE3& frameToReference_initialEstimate);
    // SE3Tracker.cpp:121-157 (lsdgpu_perma_overlap_batch, one candidate): sets and returns pointUsage
    float checkPermaRefOverlap(Frame* reference, SE3 referenceToFrame);
    // SE3Tracker.cpp:162-272 (lsdgpu_perma_track_batch, one candidate): tracks `frame` on the permaRef of `reference` and returns
    // referenceToFrame (not inverted, :271), or SE3() when it diverges.  `frame` is held active for the call; `reference` is not
    // activated: a minimized keyframe is tracked from its record and stays minimized.  Leaves numFramesTrackedOnThis and the
    // frame's pose and tracking parent alone.
    SE3 trackFrameOnPermaref(Frame* reference, Frame* frame, SE3 referenceToFrame);

    DenseDepthTrackerSettings settings;
    float pointUsage = 0, lastGoodCount = 0, lastMeanRes = 0, lastBadCount = 0, lastResidual = 0;
    float affineEstimation_a = 1, affineEstimation_b = 0;
    bool diverged = false, trackingWasGood = false;
    int mode = 1;                 // 1: device-resident LM (one kernel per frame); 0: host-driven LM

private:
    DeviceContext& dev_;
    int width_, height_;
};

// Tracking/Sim3Tracker.h:59-160 (SURVEY 8f row 1)
struct Matrix7x7 {
    float m[49];                                     // row-major
    float operator()(int r, int c) const { return m[r * 7 + c]; }
    void setZero() { for (float& v : m) v = 0.f; }
};
class Sim3Tracker {
public:
    Sim3Tracker(DeviceContext& dev, int w, int h, const Matrix3f& K);
    Sim3Tracker(const Sim3Tracker&) = delete;

    Sim3 trackFrameSim3(TrackingReference* reference, Frame* frame, const Sim3& frameToReference_initialEstimate,
                        int startLevel, int finalLevel);
    // n independent (reference, frame) pairs in one launch; members below then describe the LAST problem,
    // results[] all of them (SlamSystem::tryTrackSim3 runs two per candidate, SlamSystem.cpp:1043-1127)
    void trackFrameSim3Batch(const std::vector<TrackingReference*>& references, const std::vector<Frame*>& frames,
                             const std::vector<Sim3>& frameToReference_initialEstimates, int startLevel, int finalLevel,
                             std::vector<Sim3>& frameToReference, std::vector<lsdgpu_sim3_result>& results);

    DenseDepthTrackerSettings settings;
    Matrix7x7 lastSim3Hessian;
    float pointUsage = 0;
    float lastResidual = 0, lastDepthResidual = 0, lastPhotometricResidual = 0;
    float affineEstimation_a = 1, affineEstimation_b = 0;
    bool diverged = false;

private:
    Sim3 take(const lsdgpu_sim3_result& r);
    DeviceContext& dev_;
    int width_, height_;
};

// util/Undistorter.h:31-90: what the two camera models have in common.  Both undistort on the device of a DeviceContext.
class Undistorter {
public:
    virtual ~Undistorter() = default;
    // undistort a raw 8-bit image (in_width x in_height) on the device of `dev`, whose size must be the output size
    virtual void undistort(DeviceContext& dev, const unsigned char* image, unsigned char* result) const = 0;
    // install the tables so that Frame(dev, id, w, h, K, ts, rawImage, /*distorted=*/true) feeds raw images to the device
    virtual void install(DeviceContext& dev) const = 0;
    virtual const Matrix3f& getK() const = 0;
    virtual int getOutputWidth() const = 0;
    virtual int getOutputHeight() const = 0;
    virtual int getInputWidth() const = 0;
    virtual int getInputHeight() const = 0;
    virtual bool isValid() const = 0;
};

// Undistorter::getUndistorterForFile, util/Undistorter.cpp:38-88: 8 numbers on the first line select UndistorterOpenCV, anything
// else UndistorterPTAM; nullptr when the file cannot be read or the undistorter is invalid.  The caller owns the result.
Undistorter* getUndistorterForFile(const char* configFilename);

// util/Undistorter.h:96-160 (SURVEY 8f row 3).  The ATAN/PTAM calibration file has four lines:
//   fx fy cx cy dist   |   in_width in_height   |   "crop" / "full" / "none" / fx fy cx cy 0   |   out_width out_height
// An OpenCV-model file (8 numbers on the first line, Undistorter.cpp:70-79) is rejected here: UndistorterOpenCV reads it.
class UndistorterPTAM : public Undistorter {
public:
    explicit UndistorterPTAM(const char* configFileName);
    // undistort a raw 8-bit image (in_width x in_height) on the device of `dev`, whose size must be the output size
    void undistort(DeviceContext& dev, const unsigned char* image, unsigned char* result) const;
    // install the tables so that Frame(dev, id, w, h, K, ts, rawImage, /*distorted=*/true) feeds raw images to the device
    void install(DeviceContext& dev) const;
    const Matrix3f& getK() const { return K_; }
    int getOutputWidth() const { return out_width; }
    int getOutputHeight() const { return out_height; }
    int getInputWidth() const { return in_width; }
    int getInputHeight() const { return in_height; }
    bool isValid() const { return valid; }
    bool isPassThrough() const { return passThrough; }
    const std::vector<float>& remapTableX() const { return remapX; }
    const std::vector<float>& remapTableY() const { return remapY; }

private:
    Matrix3f K_;
    float inputCalibration[5], outputCalibration[5];
    int out_width = 0, out_height = 0, in_width = 0, in_height = 0;
    std::vector<float> remapX, remapY;
    bool valid = false, passThrough = false;
};

// util/Undistorter.h:164-239.  The OpenCV (radial-tangential) calibration file has four lines:
//   fx fy cx cy k1 k2 p1 p2   |   in_width in_height   |   "crop" / "full"   |   out_width out_height
// ("none" or explicit output parameters make it invalid, Undistorter.cpp:493-502).  The tables are built on the host without
// OpenCV (lsdgpu_undistorter_opencv_prepare, bit-identical to OpenCV 4.13's); the remap runs on the device.
class UndistorterOpenCV : public Undistorter {
public:
    explicit UndistorterOpenCV(const char* configFileName);
    void undistort(DeviceContext& dev, const unsigned char* image, unsigned char* result) const override;
    void install(DeviceContext& dev) const override;
    const Matrix3f& getK() const override { return K_; }
    int getOutputWidth() const override { return out_width; }
    int getOutputHeight() const override { return out_height; }
    int getInputWidth() const override { return in_width; }
    int getInputHeight() const override { return in_height; }
    bool isValid() const override { return valid; }
    // cv::initUndistortRectifyMap(.., CV_16SC2): (x, y) int16 pairs and the uint16 fractions, out_width*out_height each
    const std::vector<int16_t>& map1() const { return map1_; }
    const std::vector<uint16_t>& map2() const { return map2_; }

private:
    Matrix3f K_;
    float inputCalibration[8];
    int out_width = 0, out_height = 0, in_width = 0, in_height = 0;
    std::vector<int16_t> map1_;
    std::vector<uint16_t> map2_;
    bool valid = false;
};

// DepthEstimation/DepthMap.h
class DepthMap {
public:
    DepthMap(DeviceContext& dev, int w, int h, const Matrix3f& K);
    DepthMap(const DepthMap&) = delete;

    void reset();
    void updateKeyframe(std::deque<std::shared_ptr<Frame>> referenceFrames);
    void createKeyFrame(Frame* new_keyframe);
    void finalizeKeyFrame();
    void invalidate();
    bool isValid() const { return activeKeyFrame != nullptr; }
    void initializeFromGTDepth(Frame* new_frame);
    void initializeRandomly(Frame* new_frame);
    // DepthMap.cpp:920-962 from the reactivation data finalizeKeyFrame took on the device (lsdgpu_depth_set_from_existing_kf);
    // activates kf first if FrameMemory minimized it (its record keeps that data)
    void setFromExistingKF(Frame* kf);
    void setFromExistingKF(Frame* kf, const float* idepth_reAct, const float* idepthVar_reAct, const unsigned char* validity_reAct);
    // currentDepthMap in the reference's AoS layout (w*h records)
    void download(std::vector<lsdgpu_hyp>& out);

    Frame* activeKeyFrame = nullptr;

private:
    DeviceContext& dev_;
    int width_, height_;
};

}  // namespace lsd_slam
