// frame.cuh -- per-frame staging kernels: u8 -> f32 image pyramid, gradient pyramid, maxGradients,
// ground-truth depth import and the idepth / idepthVar pyramids.
//
// Replaces (paths relative to lsd_slam_core/src/):
//   Frame::Frame(.., const uchar*)        DataStructures/Frame.cpp:35-54
//   Frame::buildImage                     DataStructures/Frame.cpp:491-630
//   Frame::buildGradients                 DataStructures/Frame.cpp:643-680
//   Frame::buildMaxGradients              DataStructures/Frame.cpp:690-767
//   Frame::setDepthFromGroundTruth        DataStructures/Frame.cpp:245-293
//   Frame::buildIDepthAndIDepthVar        DataStructures/Frame.cpp:775-877
// All of these are streaming, HBM-bound passes over at most 16 B/px; the whole pyramid of one frame is built
// by ONE launch per pass (the reference builds level by level, lazily).
#pragma once
#include "internal.cuh"

// One CTA = one 16x16 level-0 tile -> 8x8, 4x4, 2x2, 1x1 on levels 1..4 (w, h are multiples of 16,
// SlamSystem.cpp:55).  The 2x2 box sum is exact in fp32 for u8-origin data (SURVEY App. A-11) and is
// associated like the scalar loop (Frame.cpp:621-624).
// SRC = PYR_PTAM fuses UndistorterPTAM::undistort (util/Undistorter.cpp:380-410) in front: level 0 is gathered bilinearly from
// the RAW (distorted) image through the remap tables, truncated to 8 bits exactly as the reference's
// `data[idx] = float expression` does, and converted to float as Frame::Frame does (Frame.cpp:44-52) -- the undistorted u8 image
// never exists in memory unless `undist` is given (parity hook / host consumers).  SRC = PYR_OPENCV does the same with
// UndistorterOpenCV's fixed-point remap (remapPixelOpenCV, maps map1 / map2, raw image in_w x in_h).
// `pitch` is the row stride of the source image in bytes: its width for the library's own staging copies, any value >= the
// width for a caller's device image (lsdgpu_frame_upload_device_u8 and its siblings; it may be odd, so loads are bytewise).
// The camera's raw pixel formats (LSDGPU_PIX_*, include/lsdgpu.h): bytes per pixel, and the 8-bit gray value of the pixel whose
// first byte is p, as cv_bridge::toCvCopy(img, MONO8) (IOWrapper/ROS/ROSImageStreamThread.cpp:117) and LiveSLAMWrapper's
// cvtColor(img, grayImg, CV_RGB2GRAY) (LiveSLAMWrapper.cpp:116-121) compute it with OpenCV 4.13: COLOR_RGB2GRAY is
// (R * 9798 + G * 19235 + B * 3735 + 2^14) >> 15 for every colour (BGR swaps R and B, the 4-channel formats ignore alpha),
// COLOR_YUV2GRAY_UYVY / _YUY2 take the luma byte of each 2-byte pixel.  Integer arithmetic, bytewise loads (the pitch may be odd).
__host__ __device__ constexpr int pixBytes(int fmt)
{
    return fmt == LSDGPU_PIX_RGB8 || fmt == LSDGPU_PIX_BGR8 ? 3 : fmt == LSDGPU_PIX_RGBA8 || fmt == LSDGPU_PIX_BGRA8 ? 4
         : fmt == LSDGPU_PIX_YUV422 || fmt == LSDGPU_PIX_YUV422_YUY2 ? 2 : 1;
}
template <int FMT>
__device__ __forceinline__ int grayOf(const uint8_t* __restrict__ p)
{
    if (FMT == LSDGPU_PIX_RGB8 || FMT == LSDGPU_PIX_RGBA8) return (__ldg(p) * 9798 + __ldg(p + 1) * 19235 + __ldg(p + 2) * 3735 + (1 << 14)) >> 15;
    if (FMT == LSDGPU_PIX_BGR8 || FMT == LSDGPU_PIX_BGRA8) return (__ldg(p + 2) * 9798 + __ldg(p + 1) * 19235 + __ldg(p) * 3735 + (1 << 14)) >> 15;
    if (FMT == LSDGPU_PIX_YUV422) return __ldg(p + 1);
    return __ldg(p);                                       // MONO8, YUV422_YUY2
}
// FMT = the raw image's pixel format: each of the four taps reads the converted value of its source pixel (conversion before the
// undistorter, as ROSImageStreamThread::vidCb orders them).  `pitch` is in bytes.
template <int FMT = LSDGPU_PIX_MONO8>
__device__ __forceinline__ unsigned char undistortPixel(const uint8_t* __restrict__ raw, int pitch, float xx, float yy)
{
    if (xx < 0) return 0;
    const int xxi = (int)xx, yyi = (int)yy;
    xx -= xxi;
    yy -= yyi;
    const float xxyy = xx * yy;
    if (FMT == LSDGPU_PIX_MONO8) {
        const uint8_t* src = raw + xxi + yyi * pitch;
        const float v = xxyy * src[1 + pitch] + (yy - xxyy) * src[pitch] + (xx - xxyy) * src[1] + (1 - xx - yy + xxyy) * src[0];
        return (unsigned char)v;
    }
    constexpr int B = pixBytes(FMT);
    const uint8_t* src = raw + xxi * B + yyi * pitch;
    const float v = xxyy * grayOf<FMT>(src + B + pitch) + (yy - xxyy) * grayOf<FMT>(src + pitch) + (xx - xxyy) * grayOf<FMT>(src + B)
                  + (1 - xx - yy + xxyy) * grayOf<FMT>(src);
    return (unsigned char)v;
}
// UndistorterOpenCV::undistort (util/Undistorter.cpp:564-567) = cv::remap(image, result, map1, map2, INTER_LINEAR) with the default
// BORDER_CONSTANT border (value 0) on u8: map1 = the integer source position (sx, sy), map2 = its 5-bit fractions (fy << 5 | fx).
// The 2x2 weights are OpenCV's 15-bit fixed-point bilinear table, (32 - fx) * (32 - fy) * 32 ... (exact, they sum to 32768); a
// tap outside the in_w x in_h image contributes 0; the sum is rounded as OpenCV's fixed-point cast, (sum + 2^14) >> 15.  Every
// tap is bounds-checked, so any pair of maps is safe to install.  FMT as for undistortPixel.
template <int FMT = LSDGPU_PIX_MONO8>
__device__ __forceinline__ unsigned char remapPixelOpenCV(const uint8_t* __restrict__ raw, int in_w, int in_h, int pitch, short2 m1,
                                                          unsigned int m2)
{
    constexpr int B = pixBytes(FMT);
    const int sx = m1.x, sy = m1.y;
    const int fx = m2 & 31, fy = (m2 >> 5) & 31;          // cv::remap reads map2 & (INTER_TAB_SIZE2 - 1)
    const bool x0 = sx >= 0 && sx < in_w, x1 = sx + 1 >= 0 && sx + 1 < in_w;
    const bool y0 = sy >= 0 && sy < in_h, y1 = sy + 1 >= 0 && sy + 1 < in_h;
    const uint8_t* s = raw + (ptrdiff_t)sy * pitch + (ptrdiff_t)sx * B;
    const int p00 = (x0 && y0) ? grayOf<FMT>(s) : 0, p01 = (x1 && y0) ? grayOf<FMT>(s + B) : 0;
    const int p10 = (x0 && y1) ? grayOf<FMT>(s + pitch) : 0, p11 = (x1 && y1) ? grayOf<FMT>(s + pitch + B) : 0;
    const int v = p00 * ((32 - fx) * (32 - fy) * 32) + p01 * (fx * (32 - fy) * 32) + p10 * ((32 - fx) * fy * 32) + p11 * (fx * fy * 32);
    return (unsigned char)((v + (1 << 14)) >> 15);
}
// source of level 0 of k_image_pyramid: the u8 image itself, or a raw image through UndistorterPTAM's / UndistorterOpenCV's tables,
// or (PYR_F32) the fp32 level 0 kept in a minimized frame's record (Frame::require after minimizeInMemory, Frame.cpp:319-338)
enum { PYR_U8 = 0, PYR_PTAM = 1, PYR_OPENCV = 2, PYR_F32 = 3 };
// src_pitch = the row stride in bytes of src (PYR_U8, PYR_PTAM, PYR_OPENCV); PYR_F32 reads w floats per row.  FMT = the pixel
// format of src (PYR_U8 with another format than MONO8 is the pass-through undistorter fed a colour or 4:2:2 camera image).
template <int SRC, int FMT = LSDGPU_PIX_MONO8>
__global__ void __launch_bounds__(256) k_image_pyramid(const uint8_t* __restrict__ src, int src_pitch, PyrPtrs p, int w, int h,
                                                       const float* __restrict__ remapX = nullptr, const float* __restrict__ remapY = nullptr,
                                                       int in_w = 0, uint8_t* __restrict__ undist = nullptr,
                                                       const short2* __restrict__ map1 = nullptr, const uint16_t* __restrict__ map2 = nullptr,
                                                       int in_h = 0)
{
    __shared__ float s0[16][17], s1[8][9], s2[4][5], s3[2][3];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int bx = blockIdx.x, by = blockIdx.y;
    const int x = bx * 16 + tx, y = by * 16 + ty;
    float v;
    if (SRC == PYR_F32)
        v = reinterpret_cast<const float*>(src)[y * w + x];
    else if (SRC != PYR_U8) {
        const unsigned char u = SRC == PYR_PTAM ? undistortPixel<FMT>(src, src_pitch, __ldg(remapX + y * w + x), __ldg(remapY + y * w + x))
                                                : remapPixelOpenCV<FMT>(src, in_w, in_h, src_pitch, map1[y * w + x], __ldg(map2 + y * w + x));
        if (undist) undist[y * w + x] = u;
        v = (float)u;
    } else if (FMT == LSDGPU_PIX_MONO8)
        v = (float)src[y * src_pitch + x];
    else
        v = (float)grayOf<FMT>(src + y * src_pitch + x * pixBytes(FMT));
    p.l[0][y * w + x] = v;
    s0[ty][tx] = v;
    __syncthreads();
    if (tx < 8 && ty < 8) {
        float a = (s0[2 * ty][2 * tx] + s0[2 * ty][2 * tx + 1] + s0[2 * ty + 1][2 * tx] + s0[2 * ty + 1][2 * tx + 1]) * 0.25f;
        s1[ty][tx] = a;
        p.l[1][(by * 8 + ty) * (w >> 1) + bx * 8 + tx] = a;
    }
    __syncthreads();
    if (tx < 4 && ty < 4) {
        float a = (s1[2 * ty][2 * tx] + s1[2 * ty][2 * tx + 1] + s1[2 * ty + 1][2 * tx] + s1[2 * ty + 1][2 * tx + 1]) * 0.25f;
        s2[ty][tx] = a;
        p.l[2][(by * 4 + ty) * (w >> 2) + bx * 4 + tx] = a;
    }
    __syncthreads();
    if (tx < 2 && ty < 2) {
        float a = (s2[2 * ty][2 * tx] + s2[2 * ty][2 * tx + 1] + s2[2 * ty + 1][2 * tx] + s2[2 * ty + 1][2 * tx + 1]) * 0.25f;
        s3[ty][tx] = a;
        p.l[3][(by * 2 + ty) * (w >> 3) + bx * 2 + tx] = a;
    }
    __syncthreads();
    if (tx == 0 && ty == 0) {
        float a = (s3[0][0] + s3[0][1] + s3[1][0] + s3[1][1]) * 0.25f;
        p.l[4][by * (w >> 4) + bx] = a;
    }
}

// Gradients of all levels in one launch (blockIdx.y = level) + maxGradients of level 0 in the same pass.
// The reference sweeps the LINEAR index range [w, w*(h-1)) so x = 0 and x = w-1 wrap across rows
// (Frame.cpp:658-677); rows 0 and h-1 are defined as zero.
// maxGradients (Frame.cpp:708-759): |grad|, then a 3x1 vertical and a 1x3 horizontal max, all over LINEAR index
// ranges, never-written cells defined as zero (SURVEY App. A-12).  |grad| is recomputed from the image for the 9
// neighbours (same fp32 operations as reading the stored gradients), which saves a launch and a pass over the
// 4.9 MB gradient level.
struct GradPtrs {
    const float* img[LSD_LEVELS];
    float4* grad[LSD_LEVELS];
    int w[LSD_LEVELS], h[LSD_LEVELS];
    float* maxgrad0;
};
__device__ __forceinline__ float absGradImg(const float* __restrict__ img, int j, int w, int h)
{
    if (j < w || j >= w * (h - 1)) return 0.f;
    const float gx = 0.5f * (__ldg(img + j + 1) - __ldg(img + j - 1));
    const float gy = 0.5f * (__ldg(img + j + w) - __ldg(img + j - w));
    return sqrtf(gx * gx + gy * gy);
}
__device__ __forceinline__ float vmax3Img(const float* __restrict__ img, int t, int w, int h)
{
    if (t < w + 1 || t >= w * (h - 1) - 1) return 0.f;
    float g1 = absGradImg(img, t - w, w, h), g2 = absGradImg(img, t, w, h), g3 = absGradImg(img, t + w, w, h);
    if (g1 < g2) g1 = g2;
    return (g1 < g3) ? g3 : g1;
}
// Level 0 is processed in 32x8 tiles (blockIdx.y == 0): |grad| of the tile + 1-cell halo is computed ONCE into shared
// memory (1.33 evaluations per pixel instead of 9), then the vertical and the horizontal 3-max run on shared memory.
// Cells are addressed by LINEAR index t = y*w + x, so the halo column x = -1 / x = w is the neighbouring row's last /
// first pixel exactly as the reference's linear sweeps see it.  Levels 1..4 (blockIdx.y = level) only need the gradient.
#define GR_TW 32
#define GR_TH 8
__global__ void __launch_bounds__(256) k_gradients(const __grid_constant__ GradPtrs p)
{
    pdlWait();                                    // launched early (programmatic dependent launch): wait for the pyramid kernel
    const int lvl = blockIdx.y;
    const int w = p.w[lvl], h = p.h[lvl];
    const float* __restrict__ img = p.img[lvl];
    if (lvl != 0) {
        const int i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= w * h) return;
        float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i >= w && i < w * (h - 1)) {
            g.x = 0.5f * (img[i + 1] - img[i - 1]);
            g.y = 0.5f * (img[i + w] - img[i - w]);
            g.z = img[i];
        }
        p.grad[lvl][i] = g;
        return;
    }
    __shared__ float ag[GR_TH + 2][GR_TW + 2];      // |grad| at linear index (y0 - 1 + r) * w + (x0 - 1 + c)
    __shared__ float vm[GR_TH][GR_TW + 2];          // vertical 3-max (Frame.cpp:721-734)
    const int tilesX = (w + GR_TW - 1) / GR_TW, tilesY = (h + GR_TH - 1) / GR_TH;
    if ((int)blockIdx.x >= tilesX * tilesY) return;
    const int x0 = (blockIdx.x % tilesX) * GR_TW, y0 = (blockIdx.x / tilesX) * GR_TH;
    const int n = w * h;
    for (int c = threadIdx.x; c < (GR_TH + 2) * (GR_TW + 2); c += 256) {
        const int cx = c % (GR_TW + 2), cy = c / (GR_TW + 2);
        const int gy = y0 - 1 + cy, gx = x0 - 1 + cx;
        float v = 0.f;
        if (gy >= 0 && gy < h && gx <= w) {
            const int t = gy * w + gx;
            if (t >= 0 && t < n) v = absGradImg(img, t, w, h);
        }
        ag[cy][cx] = v;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < GR_TH * (GR_TW + 2); c += 256) {
        const int cx = c % (GR_TW + 2), cy = c / (GR_TW + 2);
        const int gy = y0 + cy, gx = x0 - 1 + cx;
        const int t = gy * w + gx;
        float v = 0.f;
        if (gy < h && gx <= w && !(t < w + 1 || t >= w * (h - 1) - 1)) {
            float g1 = ag[cy][cx], g2 = ag[cy + 1][cx], g3 = ag[cy + 2][cx];
            if (g1 < g2) g1 = g2;
            v = (g1 < g3) ? g3 : g1;
        }
        vm[cy][cx] = v;
    }
    __syncthreads();
    const int tx = threadIdx.x % GR_TW, ty = threadIdx.x / GR_TW;
    const int x = x0 + tx, y = y0 + ty;
    if (x >= w || y >= h) return;
    const int i = y * w + x;
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i >= w && i < w * (h - 1)) {
        g.x = 0.5f * (img[i + 1] - img[i - 1]);
        g.y = 0.5f * (img[i + w] - img[i - w]);
        g.z = img[i];
    }
    p.grad[0][i] = g;
    float r;
    if (i >= w + 1 && i < w * (h - 1) - 1) {        // horizontal 3-max (Frame.cpp:740-759)
        float g1 = vm[ty][tx], g2 = vm[ty][tx + 1], g3 = vm[ty][tx + 2];
        if (g1 < g2) g1 = g2;
        r = (g1 < g3) ? g3 : g1;
    } else {
        r = (i >= w && i < w * (h - 1)) ? sqrtf(g.x * g.x + g.y * g.y) : 0.f;   // cells w and w*(h-1)-1 keep the raw |grad|
    }
    p.maxgrad0[i] = r;
}

// Frame::setDepthFromGroundTruth, Frame.cpp:264-285.  `stride` is the row stride of depth in floats: w for the library's own
// staging copy, any value >= w for a caller's device plane (lsdgpu_frame_set_depth_gt_device).
__global__ void __launch_bounds__(256) k_set_depth_gt(const float* __restrict__ depth, int stride, const float* __restrict__ maxgrad,
                                                      float* __restrict__ idepth, float* __restrict__ idepthVar,
                                                      int w, int h, float minUseGrad, float cov_scale)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w * h) return;
    const int x = i % w, y = i / w;
    const float d = depth[y * stride + x];
    if (x > 0 && x < w - 1 && y > 0 && y < h - 1 && maxgrad[i] >= minUseGrad && !isnan(d) && d > 0) {
        idepth[i] = 1.0f / d;
        idepthVar[i] = 0.01f * 0.01f * cov_scale;     // VAR_GT_INIT_INITIAL * cov_scale
    } else {
        idepth[i] = -1;
        idepthVar[i] = -1;
    }
}

// Frame::buildIDepthAndIDepthVar for levels 1..4 in one launch: one CTA = one 16x16 level-0 tile (mergeIdepth4, internal.cuh).
__global__ void __launch_bounds__(256) k_idepth_pyramid(PyrPtrs id, PyrPtrs var, int w, int h)
{
    __shared__ float2 s0[16][17], s1[8][9], s2[4][5], s3[2][3];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int bx = blockIdx.x, by = blockIdx.y;
    const int x = bx * 16 + tx, y = by * 16 + ty;
    s0[ty][tx] = make_float2(id.l[0][y * w + x], var.l[0][y * w + x]);
    __syncthreads();
    if (tx < 8 && ty < 8) {
        float2 r = mergeIdepth4(s0[2 * ty][2 * tx], s0[2 * ty][2 * tx + 1], s0[2 * ty + 1][2 * tx], s0[2 * ty + 1][2 * tx + 1]);
        s1[ty][tx] = r;
        int o = (by * 8 + ty) * (w >> 1) + bx * 8 + tx;
        id.l[1][o] = r.x; var.l[1][o] = r.y;
    }
    __syncthreads();
    if (tx < 4 && ty < 4) {
        float2 r = mergeIdepth4(s1[2 * ty][2 * tx], s1[2 * ty][2 * tx + 1], s1[2 * ty + 1][2 * tx], s1[2 * ty + 1][2 * tx + 1]);
        s2[ty][tx] = r;
        int o = (by * 4 + ty) * (w >> 2) + bx * 4 + tx;
        id.l[2][o] = r.x; var.l[2][o] = r.y;
    }
    __syncthreads();
    if (tx < 2 && ty < 2) {
        float2 r = mergeIdepth4(s2[2 * ty][2 * tx], s2[2 * ty][2 * tx + 1], s2[2 * ty + 1][2 * tx], s2[2 * ty + 1][2 * tx + 1]);
        s3[ty][tx] = r;
        int o = (by * 2 + ty) * (w >> 3) + bx * 2 + tx;
        id.l[3][o] = r.x; var.l[3][o] = r.y;
    }
    __syncthreads();
    if (tx == 0 && ty == 0) {
        float2 r = mergeIdepth4(s3[0][0], s3[0][1], s3[1][0], s3[1][1]);
        int o = by * (w >> 4) + bx;
        id.l[4][o] = r.x; var.l[4][o] = r.y;
    }
}

// UndistorterPTAM::undistort alone (u8 -> u8), util/Undistorter.cpp:380-410; `pitch` = the raw image's row stride in bytes
template <int FMT = LSDGPU_PIX_MONO8>
__global__ void __launch_bounds__(256) k_undistort(const uint8_t* __restrict__ raw, int pitch, const float* __restrict__ remapX,
                                                   const float* __restrict__ remapY, int n, uint8_t* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = undistortPixel<FMT>(raw, pitch, __ldg(remapX + i), __ldg(remapY + i));
}

// UndistorterOpenCV::undistort alone (u8 -> u8), util/Undistorter.cpp:564-567; the raw image's rows are in_w pixels apart
template <int FMT = LSDGPU_PIX_MONO8>
__global__ void __launch_bounds__(256) k_undistort_opencv(const uint8_t* __restrict__ raw, int in_w, int in_h, const short2* __restrict__ map1,
                                                          const uint16_t* __restrict__ map2, int n, uint8_t* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = remapPixelOpenCV<FMT>(raw, in_w, in_h, in_w * pixBytes(FMT), map1[i], __ldg(map2 + i));
}

// the pass-through undistorter (Undistorter.cpp:370-375) fed a colour or 4:2:2 image: cvtColor alone, w x h pixels, `pitch` bytes
// per raw row
template <int FMT>
__global__ void __launch_bounds__(256) k_to_gray(const uint8_t* __restrict__ raw, int pitch, int w, int n, uint8_t* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (uint8_t)grayOf<FMT>(raw + (i / w) * pitch + (i % w) * pixBytes(FMT));
}

// The copies of lsdgpu_frame_minimize (slot -> record) and lsdgpu_frame_activate (record -> slot): up to REC_MAX_SEGS buffers of
// a frame in one launch, 16 bytes per thread and step.  Every buffer starts 256-byte aligned and its length is rounded up to 16
// bytes (each one lies in an allocation padded to 256 bytes).
#define REC_MAX_SEGS 10
struct RecordCopy {
    const uint4* src[REC_MAX_SEGS];
    uint4* dst[REC_MAX_SEGS];
    long long end[REC_MAX_SEGS];         // cumulative length in uint4 units
    int n;
};
__global__ void __launch_bounds__(256) k_record_copy(const __grid_constant__ RecordCopy c)
{
    const long long total = c.end[c.n - 1];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int k = 0;
        while (i >= c.end[k]) k++;
        const long long o = i - (k ? c.end[k - 1] : 0);
        c.dst[k][o] = __ldg(c.src[k] + o);
    }
}
