// oracle/ref_shim/lsd_slam_viewer/keyframeGraphMsg.h -- TEST INFRASTRUCTURE.  The C++ struct roscpp generates from
// lsd_slam_viewer/msg/keyframeGraphMsg.msg (same fields, same types; boost::shared_ptr -> std::).
#pragma once
#include <cstdint>
#include <map>                  // roscpp message headers pull in <map>; KeyFrameGraphDisplay.h relies on it
#include <memory>
#include <vector>

namespace lsd_slam_viewer {
struct keyframeGraphMsg {
    uint32_t numFrames = 0;
    std::vector<uint8_t> frameData;
    uint32_t numConstraints = 0;
    std::vector<uint8_t> constraintsData;
};
typedef std::shared_ptr<keyframeGraphMsg> keyframeGraphMsgPtr;
typedef std::shared_ptr<const keyframeGraphMsg> keyframeGraphMsgConstPtr;
}
