// oracle/ref_shim/ros/package.h -- TEST INFRASTRUCTURE.  ros::package::getPath, where lsd_slam_viewer/src/KeyFrameGraphDisplay.cpp
// writes pc_tmp.ply and pc.ply: a directory the caller sets (oracle/ref_viewer_driver.cpp) instead of the ROS package path.
#pragma once
#include <string>
namespace ros {
namespace package {
inline std::string& lsdRefShimRoot() { static std::string r = "."; return r; }
inline std::string getPath(const std::string&) { return lsdRefShimRoot(); }
}
}
