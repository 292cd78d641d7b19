// lsd_host.h driven in SlamSystem's SLAM-mode order (SlamSystem.cpp): ground-truth initialisation, then per frame importFrame
// when needed, trackFrame, and updateKeyframe + clear_refPixelWasGood or, at a keyframe change, finishCurrentKeyframe
// (finalizeKeyFrame, mappingTrackingReference->importFrame, setPermaRef, invalidate) and createKeyFrame.  Every finished keyframe
// gets the constraint calls against every earlier one: checkPermaRefOverlap, trackFrameOnPermaref both ways
// (SlamSystem.cpp:1296-1305) and trackFrameSim3 both ways.  A fixed script, no decisions: used by tests/test_gpu_host_slam_mode.py.
//
//   host_slam_mode --print-globals                        the globals' values, no device touched
//   host_slam_mode --errors FRAMES                        setPermaRef / trackFrameOnPermaref misuse, one line per outcome
//   host_slam_mode FRAMES MAIN.bin CONSTRAINTS.bin [options]
//     --kf-every N            keyframe change at every frame index divisible by N (5)
//     --max-frames N          frame slots of the context (16)
//     --prune N               FrameMemory::setMaxActiveFrames(N) and pruneActiveFrames after every frame
//     --globals K g c d a s f before frame K: minUseGrad cameraPixelNoise2 depthSmoothingFactor allowNegativeIdepths
//                             useSubpixelStereo useAffineLightningEstimation
//     --reactivate K KF       before frame K: finishCurrentKeyframe, then setFromExistingKF(keyframe KF) (loadNewCurrentKeyframe)
//     --threads               the constraint calls on a second thread fed from a queue of finished keyframes
//     --device-records N      FrameMemory::setMaxDeviceRecords(N): pruneActiveFrames offloads the minimized records beyond N to
//                             host memory.  stdout also gets "MEMORY n_device device_bytes n_host host_bytes"
//                             (lsdgpu_frame_memory_usage) before setFromExistingKF and before the final DepthMap::invalidate.
//
// FRAMES: int32 w, h, n; float K[9]; float depth of frame 0 [w*h]; n images uint8 [w*h].  MAIN.bin and CONSTRAINTS.bin are raw
// records (native byte order, see put* below); stdout gets the activity of the constraint calls' reference keyframes, the
// re-activated keyframe's and the globals of the context and of a context created at the end.
#include <algorithm>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../lsd_slam_b200/host/lsd_host.h"
using namespace lsd_slam;

enum { REC_TRACK = 1, REC_KEYFRAME = 2, REC_REACTIVATE = 3, REC_FINAL = 4, REC_OVERLAP = 5, REC_PERMA = 6, REC_SIM3 = 7 };

static void putI(FILE* f, int v) { std::fwrite(&v, 4, 1, f); }
static void putF(FILE* f, float v) { std::fwrite(&v, 4, 1, f); }
static void putSE3(FILE* f, const SE3& a) { std::fwrite(a.q, 8, 4, f); std::fwrite(a.t, 8, 3, f); }
static void putSim3(FILE* f, const Sim3& a) { std::fwrite(a.q, 8, 4, f); std::fwrite(a.t, 8, 3, f); std::fwrite(&a.s, 8, 1, f); }
static void putDepth(FILE* f, DepthMap& map)
{
    std::vector<lsdgpu_hyp> h;
    map.download(h);
    std::fwrite(h.data(), sizeof(lsdgpu_hyp), h.size(), f);
}
static void putSE3Members(FILE* f, const SE3Tracker& t)
{
    for (float v : { t.pointUsage, t.lastGoodCount, t.lastMeanRes, t.lastBadCount, t.lastResidual, t.affineEstimation_a, t.affineEstimation_b })
        putF(f, v);
    putI(f, t.diverged); putI(f, t.trackingWasGood);
}

static void printGlobals(const char* what, const lsdgpu_globals& g)
{
    std::printf("%s %.9g %.9g %.9g %d %d %d\n", what, g.minUseGrad, g.cameraPixelNoise2, g.depthSmoothingFactor, g.allowNegativeIdepths,
                g.useSubpixelStereo, g.useAffineLightningEstimation);
}

struct Input {
    int w = 0, h = 0, n = 0;
    Matrix3f K;
    std::vector<float> depth0;
    std::vector<unsigned char> images;
    const unsigned char* image(int k) const { return images.data() + (size_t)k * w * h; }
};
static Input readInput(const char* path)
{
    Input in;
    FILE* f = std::fopen(path, "rb");
    if (!f) { std::perror(path); std::exit(2); }
    int hdr[3];
    bool ok = std::fread(hdr, 4, 3, f) == 3;
    in.w = hdr[0]; in.h = hdr[1]; in.n = hdr[2];
    in.depth0.resize((size_t)in.w * in.h);
    in.images.resize((size_t)in.w * in.h * in.n);
    ok = ok && std::fread(in.K.m, 4, 9, f) == 9 && std::fread(in.depth0.data(), 4, in.depth0.size(), f) == in.depth0.size() &&
         std::fread(in.images.data(), 1, in.images.size(), f) == in.images.size();
    std::fclose(f);
    if (!ok) { std::fprintf(stderr, "%s: short file\n", path); std::exit(2); }
    return in;
}

// SlamSystem's constraint thread: its own SE3Tracker and Sim3Tracker on the shared context (SlamSystem.cpp:89-90)
struct ConstraintCalls {
    ConstraintCalls(DeviceContext& dev, const Matrix3f& K, FILE* out) : se3(dev, dev.width(), dev.height(), K), sim3(dev, dev.width(), dev.height(), K), out(out) {}

    void perma(Frame* ref, Frame* fr, const SE3& init, bool report)
    {
        const bool before = ref->isActive;
        const SE3 r = se3.trackFrameOnPermaref(ref, fr, init);
        if (report) std::printf("ACTIVE perma %d %d %d\n", ref->id(), before, ref->isActive);
        putI(out, REC_PERMA); putI(out, ref->id()); putI(out, fr->id());
        putSE3(out, init); putSE3(out, r); putSE3Members(out, se3);
    }
    void trackSim3(Frame* ref, Frame* fr)
    {
        const Sim3 init = ref->getScaledCamToWorld().inverse() * fr->getScaledCamToWorld();
        TrackingReference tr;
        tr.importFrame(ref);
        const Sim3 r = sim3.trackFrameSim3(&tr, fr, init, 4, 1);
        putI(out, REC_SIM3); putI(out, ref->id()); putI(out, fr->id());
        putSim3(out, init); putSim3(out, r);
        for (float v : { sim3.pointUsage, sim3.lastResidual, sim3.lastDepthResidual, sim3.lastPhotometricResidual, sim3.affineEstimation_a,
                         sim3.affineEstimation_b })
            putF(out, v);
        putI(out, sim3.diverged);
        std::fwrite(sim3.lastSim3Hessian.m, 4, 49, out);
    }
    // a newly finished keyframe against every keyframe finished before it
    void process(Frame* kf)
    {
        for (Frame* c : finished) {
            const SE3 c2f = se3FromSim3(kf->getScaledCamToWorld().inverse() * c->getScaledCamToWorld());
            const bool before = c->isActive;
            const float usage = se3.checkPermaRefOverlap(c, c2f);
            std::printf("ACTIVE overlap %d %d %d\n", c->id(), before, c->isActive);
            putI(out, REC_OVERLAP); putI(out, c->id()); putI(out, kf->id()); putSE3(out, c2f); putF(out, usage); putF(out, se3.pointUsage);
            perma(c, kf, c2f, true);
            perma(kf, c, c2f.inverse(), false);
            trackSim3(c, kf);
            trackSim3(kf, c);
        }
        finished.push_back(kf);
        std::fflush(stdout);
    }

    SE3Tracker se3;
    Sim3Tracker sim3;
    FILE* out;
    std::vector<Frame*> finished;
};

// the queue of SlamSystem::newKeyFrames and the thread that drains it (SlamSystem::constraintSearchThreadLoop)
struct ConstraintThread {
    explicit ConstraintThread(ConstraintCalls& calls) : calls(calls), worker([this] { run(); }) {}
    ~ConstraintThread()
    {
        if (!worker.joinable()) return;
        { std::lock_guard<std::mutex> l(mu); stop = true; cv.notify_one(); }
        worker.join();
    }
    void push(Frame* kf)
    {
        std::lock_guard<std::mutex> l(mu);
        queue.push_back(kf);
        cv.notify_one();
    }
    void finish()
    {
        { std::lock_guard<std::mutex> l(mu); stop = true; cv.notify_one(); }
        worker.join();
        if (!error.empty()) throw LsdGpuError(error);
    }
    void run()
    {
        for (;;) {
            Frame* kf;
            {
                std::unique_lock<std::mutex> l(mu);
                cv.wait(l, [this] { return stop || !queue.empty(); });
                if (queue.empty()) return;
                kf = queue.front();
                queue.pop_front();
            }
            try { calls.process(kf); } catch (const std::exception& e) { std::lock_guard<std::mutex> l(mu); error = e.what(); return; }
        }
    }

    ConstraintCalls& calls;
    std::mutex mu;
    std::condition_variable cv;
    std::deque<Frame*> queue;
    bool stop = false;
    std::string error;
    std::thread worker;
};

static int runErrors(const Input& in)
{
    DeviceContext dev(0, in.w, in.h, in.K, 4);
    Frame f0(dev, 0, in.w, in.h, in.K, 0, in.image(0)), f1(dev, 1, in.w, in.h, in.K, 1, in.image(1));
    std::vector<float> d1(in.depth0);
    for (float& v : d1) v *= 2;
    f0.setDepthFromGroundTruth(in.depth0.data());
    f1.setDepthFromGroundTruth(d1.data());
    TrackingReference r0, r1;
    r0.importFrame(&f0);
    r1.importFrame(&f1);
    SE3Tracker t(dev, in.w, in.h, in.K);
    SE3 pose;
    pose.t[0] = 0.3; pose.t[2] = -0.2;
    f0.setPermaRef(&r0);
    const int n0 = f0.permaRefNumPts;
    const float u0 = t.checkPermaRefOverlap(&f0, pose);
    try {
        f0.setPermaRef(&r1);
        std::printf("setPermaRef no error\n");
    } catch (const LsdGpuError& e) {
        std::printf("setPermaRef error %s\n", e.what());
    }
    const float u1 = t.checkPermaRefOverlap(&f0, pose);
    try {
        t.trackFrameOnPermaref(&f1, &f0, pose);
        std::printf("trackFrameOnPermaref no error\n");
    } catch (const LsdGpuError& e) {
        std::printf("trackFrameOnPermaref error %s\n", e.what());
    }
    f1.setPermaRef(&r1);                                       // what the rejected call would have frozen
    const float u2 = t.checkPermaRefOverlap(&f1, pose);
    std::printf("permaRef %d %d %.9g %.9g %d %.9g\n", n0, f0.permaRefNumPts, u0, u1, f1.permaRefNumPts, u2);
    return 0;
}

int main(int argc, char** argv)
{
    if (argc >= 2 && std::strcmp(argv[1], "--print-globals") == 0) {
        lsdgpu_globals g;
        g.minUseGrad = minUseGrad; g.cameraPixelNoise2 = cameraPixelNoise2; g.depthSmoothingFactor = depthSmoothingFactor;
        g.allowNegativeIdepths = allowNegativeIdepths; g.useSubpixelStereo = useSubpixelStereo;
        g.useAffineLightningEstimation = useAffineLightningEstimation;
        printGlobals("globals", g);
        return 0;
    }
    if (argc >= 3 && std::strcmp(argv[1], "--errors") == 0) return runErrors(readInput(argv[2]));
    if (argc < 4) { std::fprintf(stderr, "usage: see the head of host_slam_mode.cpp\n"); return 2; }
    const Input in = readInput(argv[1]);
    int kfEvery = 5, maxFrames = 16, prune = -1, globalsAt = -1, reactAt = -1, reactKf = -1;
    bool threads = false, deviceRecordsSet = false;
    int deviceRecords = -1;
    float gf[3] = { 0, 0, 0 };
    int gb[3] = { 0, 0, 0 };
    for (int i = 4; i < argc; i++) {
        const std::string a = argv[i];
        if (a == "--kf-every") kfEvery = std::atoi(argv[++i]);
        else if (a == "--max-frames") maxFrames = std::atoi(argv[++i]);
        else if (a == "--prune") prune = std::atoi(argv[++i]);
        else if (a == "--threads") threads = true;
        else if (a == "--device-records") { deviceRecords = std::atoi(argv[++i]); deviceRecordsSet = true; }
        else if (a == "--reactivate") { reactAt = std::atoi(argv[i + 1]); reactKf = std::atoi(argv[i + 2]); i += 2; }
        else if (a == "--globals") {
            globalsAt = std::atoi(argv[++i]);
            for (float& v : gf) v = (float)std::atof(argv[++i]);
            for (int& v : gb) v = std::atoi(argv[++i]);
        } else { std::fprintf(stderr, "unknown option %s\n", a.c_str()); return 2; }
    }
    FILE* out = std::fopen(argv[2], "wb");
    FILE* cons = std::fopen(argv[3], "wb");
    if (!out || !cons) { std::perror("output"); return 2; }

    try {
        DeviceContext dev(0, in.w, in.h, in.K, maxFrames);
        if (prune >= 0) dev.frameMemory().setMaxActiveFrames(prune);
        if (deviceRecordsSet) dev.frameMemory().setMaxDeviceRecords(deviceRecords);
        auto reportMemory = [&] {
            if (!deviceRecordsSet) return;
            int nd = 0, nh = 0;
            size_t db = 0, hb = 0;
            dev.check(lsdgpu_frame_memory_usage(dev.raw(), &nd, &db, &nh, &hb), "lsdgpu_frame_memory_usage");
            std::printf("MEMORY %d %zu %d %zu\n", nd, db, nh, hb);
        };
        SE3Tracker tracker(dev, in.w, in.h, in.K);
        for (int lvl = 4; lvl < LSDGPU_LEVELS; lvl++) tracker.settings.maxItsPerLvl[lvl] = 0;     // SlamSystem.cpp:80-81
        DepthMap map(dev, in.w, in.h, in.K);
        TrackingReference trackingReference, mappingTrackingReference;
        std::map<int, std::unique_ptr<Frame>> keyframes;         // outlive the constraint thread
        std::vector<int> keyframeOrder;                          // keyframesAll: a keyframe is listed once, when first finished
        ConstraintCalls calls(dev, in.K, cons);
        std::unique_ptr<ConstraintThread> thread(threads ? new ConstraintThread(calls) : nullptr);

        // gtDepthInit (SlamSystem.cpp:830-852)
        std::unique_ptr<Frame> prev(new Frame(dev, 0, in.w, in.h, in.K, 0, in.image(0)));
        prev->setDepthFromGroundTruth(in.depth0.data());
        map.initializeFromGTDepth(prev.get());
        Frame* current = prev.get();
        keyframes[0] = std::move(prev);
        Frame* last = current;
        std::unique_ptr<Frame> lastOwned;

        auto finishCurrentKeyframe = [&] {                       // SlamSystem.cpp:396-420
            map.finalizeKeyFrame();
            mappingTrackingReference.importFrame(current);
            current->setPermaRef(&mappingTrackingReference);
            mappingTrackingReference.invalidate();
            const bool first = std::find(keyframeOrder.begin(), keyframeOrder.end(), current->id()) == keyframeOrder.end();
            if (!first) return;
            keyframeOrder.push_back(current->id());
            if (thread) thread->push(current);
        };
        auto constraintsInline = [&](Frame* kf) { if (!thread && kf) calls.process(kf); };

        for (int k = 1; k < in.n; k++) {
            if (k == globalsAt) {
                minUseGrad = gf[0]; cameraPixelNoise2 = gf[1]; depthSmoothingFactor = gf[2];
                allowNegativeIdepths = gb[0] != 0; useSubpixelStereo = gb[1] != 0; useAffineLightningEstimation = gb[2] != 0;
            }
            if (k == reactAt) {                                  // changeKeyframe with an old keyframe (SlamSystem.cpp:491-500)
                Frame* old = current;
                const size_t before = keyframeOrder.size();
                finishCurrentKeyframe();
                Frame* kf = keyframes.at(reactKf).get();
                std::printf("REACTIVATE %d %d\n", kf->id(), kf->isActive);
                reportMemory();
                map.setFromExistingKF(kf);
                current = kf;
                putI(out, REC_REACTIVATE); putI(out, old->id()); putI(out, kf->id()); putI(out, old->permaRefNumPts);
                putDepth(out, map);
                constraintsInline(keyframeOrder.size() > before ? old : nullptr);
            }
            std::unique_ptr<Frame> frame(new Frame(dev, k, in.w, in.h, in.K, k, in.image(k)));
            if (trackingReference.keyframe != current || current->depthHasBeenUpdatedFlag())   // SlamSystem.cpp:907-912
                trackingReference.importFrame(current);
            const SE3 init = se3FromSim3(current->getScaledCamToWorld().inverse() * last->getScaledCamToWorld());   // :922-923
            const SE3 pose = tracker.trackFrame(&trackingReference, frame.get(), init);
            putI(out, REC_TRACK); putI(out, k); putI(out, current->id());
            putSE3(out, init); putSE3(out, pose); putSE3Members(out, tracker);
            if (tracker.diverged) throw LsdGpuError("frame " + std::to_string(k) + " diverged");
            lastOwned.reset();                                   // the previous frame's pose was the last one read
            last = frame.get();
            if (k % kfEvery == 0) {
                Frame* old = current;
                const size_t before = keyframeOrder.size();
                finishCurrentKeyframe();
                map.createKeyFrame(frame.get());
                current = frame.get();
                putI(out, REC_KEYFRAME); putI(out, old->id()); putI(out, k); putI(out, old->permaRefNumPts);
                putSim3(out, frame->pose->thisToParent_raw);
                putDepth(out, map);
                keyframes[k] = std::move(frame);
                constraintsInline(keyframeOrder.size() > before ? old : nullptr);
            } else {
                std::deque<std::shared_ptr<Frame>> refs;
                refs.push_back(std::shared_ptr<Frame>(frame.get(), [](Frame*) {}));
                map.updateKeyframe(refs);
                frame->clear_refPixelWasGood();
                lastOwned = std::move(frame);
            }
            if (prune >= 0) dev.frameMemory().pruneActiveFrames();
        }
        if (thread) thread->finish();
        putI(out, REC_FINAL);
        putDepth(out, map);
        lsdgpu_globals g;
        dev.check(lsdgpu_get_globals(dev.raw(), &g), "lsdgpu_get_globals");
        printGlobals("context", g);
        {
            DeviceContext fresh(0, in.w, in.h, in.K, 2);
            fresh.check(lsdgpu_get_globals(fresh.raw(), &g), "lsdgpu_get_globals");
            printGlobals("fresh", g);
        }
        lastOwned.reset();
        reportMemory();
        map.invalidate();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    std::fclose(out);
    std::fclose(cons);
    return 0;
}
