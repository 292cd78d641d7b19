/* colour_input_oracle.c -- plain-C restatement of the gray conversion in front of the undistorter for the tests:
 * cv_bridge::toCvCopy(img, MONO8) (IOWrapper/ROS/ROSImageStreamThread.cpp:117) and LiveSLAMWrapper::newImageCallback's
 * cvtColor(img, grayImg, CV_RGB2GRAY) (LiveSLAMWrapper.cpp:116-121), as OpenCV 4.13's cv::cvtColor computes them on 8-bit images:
 *   COLOR_RGB2GRAY   (R * 9798 + G * 19235 + B * 3735 + (1 << 14)) >> 15   (the weights are 0.299, 0.587, 0.114 in 15-bit fixed
 *                    point; RGBA ignores alpha)
 *   COLOR_BGR2GRAY   the same with R and B swapped
 *   COLOR_YUV2GRAY_UYVY / _YUY2   the luma byte of each 2-byte pixel: byte 1 / byte 0
 * Test infrastructure only: written apart from the library (lsd_slam_b200/csrc/frame.cuh), never linked into it.  The format
 * numbers are include/lsdgpu.h's LSDGPU_PIX_*.  Build: cc -O2 -shared -fPIC. */
#include <stddef.h>
#include <stdint.h>

int lsdo_cvt_bytes_per_pixel(int fmt)
{
    switch (fmt) {
    case 0: return 1;                 /* mono8 */
    case 1: case 2: return 3;         /* rgb8, bgr8 */
    case 3: case 4: return 4;         /* rgba8, bgra8 */
    case 5: case 6: return 2;         /* yuv422 (UYVY), yuv422_yuy2 */
    default: return 0;
    }
}

static int rgb_to_gray(int r, int g, int b)
{
    return (r * 9798 + g * 19235 + b * 3735 + (1 << 14)) >> 15;
}

/* raw (h rows of `pitch` bytes, w pixels of format fmt) -> out (w * h bytes); returns -1 for an unknown format */
int lsdo_cvt_gray(int fmt, const uint8_t* raw, int w, int h, size_t pitch, uint8_t* out)
{
    const int bpp = lsdo_cvt_bytes_per_pixel(fmt);
    if (!bpp) return -1;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const uint8_t* p = raw + (size_t)y * pitch + (size_t)x * bpp;
            int v;
            if (fmt == 1 || fmt == 3) v = rgb_to_gray(p[0], p[1], p[2]);
            else if (fmt == 2 || fmt == 4) v = rgb_to_gray(p[2], p[1], p[0]);
            else if (fmt == 5) v = p[1];
            else v = p[0];
            out[(size_t)y * w + x] = (uint8_t)v;
        }
    return 0;
}

/* the gray value of every 24-bit colour, indexed by R << 16 | G << 8 | B (2^24 bytes) */
void lsdo_cvt_rgb_table(uint8_t* out)
{
    for (int c = 0; c < (1 << 24); c++) out[c] = (uint8_t)rgb_to_gray(c >> 16, (c >> 8) & 255, c & 255);
}
