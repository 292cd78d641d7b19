// output.cuh -- what leaves the path when a keyframe is finished (SURVEY 8f row 4), packed on the device so that the
// keyframe crosses PCIe once, in wire layout.
//
// Replaces (paths relative to lsd_slam_core/src/):
//   ROSOutput3DWrapper::publishKeyframe, packing loop   IOWrapper/ROS/ROSOutput3DWrapper.cpp:91-110
//       InputPointDense {float idepth; float idepth_var; uchar color[4];}   IOWrapper/ROS/ROSOutput3DWrapper.h:34-39
//       (= lsd_slam_viewer/msg/keyframeMsg.msg:20-22 `uint8[] pointcloud`, 12 bytes per pixel of the publish level)
#pragma once
#include "internal.cuh"

// One thread per 32-bit WORD of the packed cloud (3 words per pixel): stores are perfectly coalesced, the three
// source planes are read through L1/L2 (each value is needed by at most two neighbouring threads).
__global__ void __launch_bounds__(256) k_pack_pointcloud(const float* __restrict__ idepth, const float* __restrict__ idepthVar,
                                                         const float* __restrict__ color, int n, uint32_t* __restrict__ out)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= 3 * n) return;
    const int px = j / 3, part = j - 3 * px;
    uint32_t v;
    if (part == 0) v = __float_as_uint(__ldg(idepth + px));
    else if (part == 1) v = __float_as_uint(__ldg(idepthVar + px));
    else {
        const uint32_t c = (uint32_t)(unsigned char)__ldg(color + px);      // float -> uchar conversion of the reference (:103-106)
        v = c * 0x01010101u;
    }
    out[j] = v;
}
