// oracle/ref_shim/lsd_slam_viewer/keyframeMsg.h -- TEST INFRASTRUCTURE.  The C++ struct roscpp generates from
// lsd_slam_viewer/msg/keyframeMsg.msg (same fields, same types; boost::array / boost::shared_ptr -> std::).
#pragma once
#include <array>
#include <cstdint>
#include <memory>
#include <vector>

namespace lsd_slam_viewer {
struct keyframeMsg {
    int32_t id = 0;
    double time = 0;
    uint8_t isKeyframe = 0;
    std::array<float, 7> camToWorld{};
    float fx = 0, fy = 0, cx = 0, cy = 0;
    uint32_t height = 0, width = 0;
    std::vector<uint8_t> pointcloud;
};
typedef std::shared_ptr<keyframeMsg> keyframeMsgPtr;
typedef std::shared_ptr<const keyframeMsg> keyframeMsgConstPtr;
}
