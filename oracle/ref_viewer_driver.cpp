// oracle/ref_viewer_driver.cpp -- TEST INFRASTRUCTURE.  Drives lsd_slam_viewer's own KeyFrameDisplay (compiled unmodified by
// oracle/cloud.py into oracle/_ref/libviewer_ref.so, against the stand-ins of oracle/ref_shim) the way the viewer does for one
// keyframe: a keyframeMsg through setFrom (KeyFrameDisplay.cpp:65-104), refreshPC (:106-222) with the filter settings as the
// viewer's globals (settings.cpp:36-40), then flushPC (:269-339) into a file.  Exports the vertex buffer refreshPC hands to
// glBufferData, the flushed bytes and totalPoints / displayedPoints; and, for a whole map, the pc.ply KeyFrameGraphDisplay writes.
#include <cstdio>
#include <cstring>
#include <fstream>
#include <vector>

#include "KeyFrameDisplay.h"
#include "KeyFrameGraphDisplay.h"
#include "settings.h"
#include "ros/package.h"

extern "C" int lsdv_ref_keyframe(const unsigned char* pointcloud, int width, int height, float fx, float fy, float cx, float cy,
                                 const float camToWorld[7], float scaledTH, float absTH, int nearSupport, const char* tmp_path,
                                 void* vertex_out, void* ply_out, int* total, int* displayed)
{
    scaledDepthVarTH = scaledTH;
    absDepthVarTH = absTH;
    minNearSupport = nearSupport;
    sparsifyFactor = 1;
    keepInMemory = true;

    auto msg = std::make_shared<lsd_slam_viewer::keyframeMsg>();
    memcpy(msg->camToWorld.data(), camToWorld, 7 * sizeof(float));
    msg->fx = fx; msg->fy = fy; msg->cx = cx; msg->cy = cy;
    msg->width = (uint32_t)width; msg->height = (uint32_t)height;
    msg->pointcloud.assign(pointcloud, pointcloud + (size_t)width * height * sizeof(InputPointDense));

    KeyFrameDisplay* d = new KeyFrameDisplay();
    d->setFrom(msg);
    d->refreshPC();
    const std::vector<unsigned char>& vb = lsd_ref_shim_gl::lastBuffer();
    if (vertex_out && !vb.empty()) memcpy(vertex_out, vb.data(), vb.size());
    *total = d->totalPoints;
    *displayed = d->displayedPoints;

    int num;
    {
        std::ofstream f(tmp_path, std::ios::binary);
        num = d->flushPC(&f);
    }
    if (ply_out && num > 0) {
        FILE* fp = fopen(tmp_path, "rb");
        if (!fp) { delete d; return -1; }
        size_t got = fread(ply_out, 1, (size_t)num * 16, fp);
        fclose(fp);
        if (got != (size_t)num * 16) { delete d; return -1; }
    }
    remove(tmp_path);
    delete d;
    return num;
}

// The viewer's "save pc.ply" path for a whole map, KeyFrameGraphDisplay.cpp:60-92: every keyframe through addMsg (:127-141), then
// draw() with flushPointcloud set and cutFirstNKf = -1 (all keyframes), which writes <dir>/pc.ply.  pointclouds = n records of
// width*height InputPointDense each, camToWorld = 7 floats per keyframe.  Returns 0.
extern "C" int lsdv_ref_map_ply(int n, const unsigned char* pointclouds, int width, int height, float fx, float fy, float cx, float cy,
                                const float* camToWorld, float scaledTH, float absTH, int nearSupport, const char* dir)
{
    scaledDepthVarTH = scaledTH;
    absDepthVarTH = absTH;
    minNearSupport = nearSupport;
    sparsifyFactor = 1;
    keepInMemory = true;
    cutFirstNKf = -1;
    ros::package::lsdRefShimRoot() = dir;
    const size_t bytes = (size_t)width * height * sizeof(InputPointDense);
    KeyFrameGraphDisplay* g = new KeyFrameGraphDisplay();
    for (int i = 0; i < n; i++) {
        auto msg = std::make_shared<lsd_slam_viewer::keyframeMsg>();
        msg->id = i;
        memcpy(msg->camToWorld.data(), camToWorld + 7 * (size_t)i, 7 * sizeof(float));
        msg->fx = fx; msg->fy = fy; msg->cx = cx; msg->cy = cy;
        msg->width = (uint32_t)width; msg->height = (uint32_t)height;
        msg->pointcloud.assign(pointclouds + i * bytes, pointclouds + (i + 1) * bytes);
        g->addMsg(msg);
    }
    g->flushPointcloud = true;
    g->draw();
    delete g;
    return 0;
}
