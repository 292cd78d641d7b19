// host_slam_mode.cpp's SLAM-mode script, unchanged, with FrameMemory::setMaxDeviceRecords(N) on every DeviceContext it creates: each
// pruneActiveFrames then offloads the minimized records beyond N to host memory (lsdgpu_frame_offload).  Used by
// tests/test_gpu_host_offload.py.
//
//   host_slam_mode_offload FRAMES MAIN.bin CONSTRAINTS.bin --device-records N [host_slam_mode's options]
//
// Besides host_slam_mode's output, stdout gets "MEMORY n_device device_bytes n_host host_bytes" (lsdgpu_frame_memory_usage) right
// before DepthMap::setFromExistingKF and before the final DepthMap::invalidate.
//
// The script's DeviceContext and DepthMap are replaced by the subclasses below, by name, so that the script itself is not repeated.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../lsd_slam_b200/host/lsd_host.h"

namespace {
int deviceRecords = -1;

class OffloadDeviceContext : public lsd_slam::DeviceContext {
public:
    OffloadDeviceContext(int device, int w, int h, const lsd_slam::Matrix3f& K, int maxFrames)
        : lsd_slam::DeviceContext(device, w, h, K, maxFrames)
    {
        frameMemory().setMaxDeviceRecords(deviceRecords);
    }
};

class MemoryReportingDepthMap : public lsd_slam::DepthMap {
public:
    MemoryReportingDepthMap(lsd_slam::DeviceContext& dev, int w, int h, const lsd_slam::Matrix3f& K)
        : lsd_slam::DepthMap(dev, w, h, K), dev_(dev) {}
    using lsd_slam::DepthMap::setFromExistingKF;
    void setFromExistingKF(lsd_slam::Frame* kf)
    {
        report();
        lsd_slam::DepthMap::setFromExistingKF(kf);
    }
    void invalidate()
    {
        report();
        lsd_slam::DepthMap::invalidate();
    }

private:
    void report() const
    {
        int nd = 0, nh = 0;
        size_t db = 0, hb = 0;
        dev_.check(lsdgpu_frame_memory_usage(dev_.raw(), &nd, &db, &nh, &hb), "lsdgpu_frame_memory_usage");
        std::printf("MEMORY %d %zu %d %zu\n", nd, db, nh, hb);
    }
    lsd_slam::DeviceContext& dev_;
};
}  // namespace

#define DeviceContext OffloadDeviceContext
#define DepthMap MemoryReportingDepthMap
#define main host_slam_mode_main
#include "host_slam_mode.cpp"
#undef main

int main(int argc, char** argv)
{
    std::vector<char*> args;                             // host_slam_mode's arguments: all but --device-records N
    for (int i = 0; i < argc; i++) {
        if (std::strcmp(argv[i], "--device-records") == 0 && i + 1 < argc) deviceRecords = std::atoi(argv[++i]);
        else args.push_back(argv[i]);
    }
    if (deviceRecords < 0) { std::fprintf(stderr, "usage: see the head of host_slam_mode_offload.cpp\n"); return 2; }
    args.push_back(nullptr);
    return host_slam_mode_main((int)args.size() - 1, args.data());
}
