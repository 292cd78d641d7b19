/* undistort_opencv_oracle.c -- plain-C restatement of UndistorterOpenCV (util/Undistorter.cpp:449-567) for the tests: the table
 * builder (cv::getOptimalNewCameraMatrix + cv::initUndistortRectifyMap(.., CV_16SC2) as OpenCV 4.13 computes them for the
 * 4-coefficient model) and cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) on u8.  Test infrastructure only: written apart from the
 * library (lsd_slam_b200/csrc/frames.cu, frame.cuh), never linked into it.  Build: cc -O2 -ffp-contract=off -shared -fPIC. */
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>

/* cvRound(double): nearest, ties to even; outside the int range INT_MIN (cvtsd2si) */
static int round_even(double v)
{
    if (!(v > -2147483648.5 && v < 2147483647.5)) return INT_MIN;
    return (int)nearbyint(v);
}

static short sat16(int v)
{
    if (v < SHRT_MIN) return SHRT_MIN;
    if (v > SHRT_MAX) return SHRT_MAX;
    return (short)v;
}

/* undistortPoints, default criteria (5 iterations, no epsilon), one point; OpenCV 4.x resets to the raw ray when icdist < 0 */
static void undistort_point(double u, double v, const double K[4], const double D[4], double* ox, double* oy)
{
    const double fx = K[0], fy = K[1], cx = K[2], cy = K[3];
    const double ifx = 1. / fx, ify = 1. / fy;
    double x = (u - cx) * ifx, y = (v - cy) * ify;
    const double x0 = x, y0 = y;
    int it;
    for (it = 0; it < 5; it++) {
        double r2 = x * x + y * y;
        double icdist = 1 / (1 + (D[1] * r2 + D[0]) * r2);
        double dx, dy;
        if (icdist < 0) {
            x = (u - cx) * ifx;
            y = (v - cy) * ify;
            break;
        }
        dx = 2 * D[2] * x * y + D[3] * (r2 + 2 * x * x);
        dy = D[2] * (r2 + 2 * y * y) + 2 * D[3] * x * y;
        x = (x0 - dx) * icdist;
        y = (y0 - dy) * icdist;
    }
    *ox = x;
    *oy = y;
}

static void map_entry(double X, double Y, double W, const double K[4], const double D[4], short* m1, unsigned short* m2)
{
    double w = 1. / W, x = X * w, y = Y * w;
    double x2 = x * x, y2 = y * y, r2 = x2 + y2, xy2 = 2 * x * y;
    double kr = 1 + (D[1] * r2 + D[0]) * r2;
    double xd = x * kr + D[2] * xy2 + D[3] * (r2 + 2 * x2);
    double yd = y * kr + D[2] * (r2 + 2 * y2) + D[3] * xy2;
    int iu = round_even((K[0] * xd + K[2]) * 32.0);
    int iv = round_even((K[1] * yd + K[3]) * 32.0);
    m1[0] = sat16(iu >> 5);
    m1[1] = sat16(iv >> 5);
    *m2 = (unsigned short)((iv & 31) * 32 + (iu & 31));
}

/* mode -1 "crop" (alpha 0), -2 "full" (alpha 1).  Returns 0, or -2 when invalid. */
int lsdo_cv_prepare(const float calib[8], int in_w, int in_h, int mode, int out_w, int out_h,
                    short* map1, unsigned short* map2, double Knew[9], float Kout[9])
{
    float c[8];
    double K[4], D[4], alpha, px[81], py[81];
    double inX0 = -FLT_MAX, inX1 = FLT_MAX, inY0 = -FLT_MAX, inY1 = FLT_MAX;
    double outX0 = FLT_MAX, outX1 = -FLT_MAX, outY0 = FLT_MAX, outY1 = -FLT_MAX;
    double f0x, f0y, c0x, c0y, f1x, f1y, c1x, c1y, A[9], det, id, inv[9];
    int i, j, k;
    if (in_w <= 0 || in_h <= 0 || out_w <= 0 || out_h <= 0 || (mode != -1 && mode != -2)) return -2;
    for (i = 0; i < 8; i++) c[i] = calib[i];
    if (c[2] < 1.0f) {                 /* Undistorter.cpp:519-534 */
        c[0] = c[0] * in_w; c[2] = c[2] * in_w;
        c[1] = c[1] * in_h; c[3] = c[3] * in_h;
    }
    K[0] = c[0]; K[1] = c[1]; K[2] = c[2]; K[3] = c[3];
    for (i = 0; i < 4; i++) D[i] = c[4 + i];
    alpha = mode == -2 ? 1.0 : 0.0;

    /* getOptimalNewCameraMatrix: 9x9 grid over [0, w-1] x [0, h-1]; inner = the sides' innermost, outer = border bounding box */
    for (j = 0; j < 9; j++)
        for (i = 0; i < 9; i++)
            undistort_point((double)i * (in_w - 1) / 8, (double)j * (in_h - 1) / 8, K, D, &px[j * 9 + i], &py[j * 9 + i]);
    for (j = 0; j < 9; j++)
        for (i = 0; i < 9; i++) {
            double x = px[j * 9 + i], y = py[j * 9 + i];
            if (i == 0 || i == 8 || j == 0 || j == 8) {
                if (x < outX0) outX0 = x;
                if (outX1 < x) outX1 = x;
                if (y < outY0) outY0 = y;
                if (outY1 < y) outY1 = y;
            }
            if (i == 0 && inX0 < x) inX0 = x;
            if (i == 8 && x < inX1) inX1 = x;
            if (j == 0 && inY0 < y) inY0 = y;
            if (j == 8 && y < inY1) inY1 = y;
        }
    f0x = (out_w - 1) / (inX1 - inX0); f0y = (out_h - 1) / (inY1 - inY0);
    c0x = -f0x * inX0; c0y = -f0y * inY0;
    f1x = (out_w - 1) / (outX1 - outX0); f1y = (out_h - 1) / (outY1 - outY0);
    c1x = -f1x * outX0; c1y = -f1y * outY0;
    for (i = 0; i < 9; i++) A[i] = 0;
    A[0] = f0x * (1 - alpha) + f1x * alpha;
    A[2] = c0x * (1 - alpha) + c1x * alpha;
    A[4] = f0y * (1 - alpha) + f1y * alpha;
    A[5] = c0y * (1 - alpha) + c1y * alpha;
    A[8] = 1;
    if (Knew) for (i = 0; i < 9; i++) Knew[i] = A[i];
    if (Kout) {                        /* getK() is K_ transposed (:557); main_on_images.cpp:164-167 reads (0,0) (1,1) (2,0) (2,1) */
        for (i = 0; i < 9; i++) Kout[i] = 0;
        Kout[0] = (float)A[0]; Kout[4] = (float)A[4];
        Kout[2] = (float)A[2]; Kout[5] = (float)A[5];
        Kout[8] = 1;
    }
    if (!map1 || !map2) return 0;

    /* initUndistortRectifyMap: the inverse of A by 3x3 cofactors / det, rows walked as OpenCV's AVX2 loop does */
    det = A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
    if (det == 0) return -2;
    id = 1. / det;
    inv[0] = (A[4] * A[8] - A[5] * A[7]) * id; inv[1] = (A[2] * A[7] - A[1] * A[8]) * id; inv[2] = (A[1] * A[5] - A[2] * A[4]) * id;
    inv[3] = (A[5] * A[6] - A[3] * A[8]) * id; inv[4] = (A[0] * A[8] - A[2] * A[6]) * id; inv[5] = (A[2] * A[3] - A[0] * A[5]) * id;
    inv[6] = (A[3] * A[7] - A[4] * A[6]) * id; inv[7] = (A[1] * A[6] - A[0] * A[7]) * id; inv[8] = (A[0] * A[4] - A[1] * A[3]) * id;
    for (j = 0; j < out_h; j++) {
        double rx = j * inv[1] + inv[2], ry = j * inv[4] + inv[5], rw = j * inv[7] + inv[8];
        short* m1 = map1 + (long)2 * j * out_w;
        unsigned short* m2 = map2 + (long)j * out_w;
        for (i = 0; i + 8 <= out_w; i += 8) {
            for (k = 0; k < 8; k++)
                map_entry(rx + k * inv[0], ry + k * inv[3], rw + k * inv[6], K, D, m1 + 2 * (i + k), m2 + i + k);
            rx += 8 * inv[0]; ry += 8 * inv[3]; rw += 8 * inv[6];
        }
        for (; i < out_w; i++) {
            map_entry(rx, ry, rw, K, D, m1 + 2 * i, m2 + i);
            rx += inv[0]; ry += inv[3]; rw += inv[6];
        }
    }
    return 0;
}

/* cv::remap(src, dst, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) for 8-bit single-channel images */
void lsdo_cv_remap(const uint8_t* src, int in_w, int in_h, const short* map1, const unsigned short* map2, int out_w, int out_h,
                   uint8_t* dst)
{
    long n = (long)out_w * out_h, p;
    for (p = 0; p < n; p++) {
        int sx = map1[2 * p], sy = map1[2 * p + 1];
        int a = map2[p] & 1023, fx = a & 31, fy = a >> 5;
        int w00 = (32 - fx) * (32 - fy) * 32, w01 = fx * (32 - fy) * 32, w10 = (32 - fx) * fy * 32, w11 = fx * fy * 32;
        int v00, v01, v10, v11;
        if (sx >= in_w || sx + 1 < 0 || sy >= in_h || sy + 1 < 0) { dst[p] = 0; continue; }
        v00 = (sx >= 0 && sy >= 0) ? src[(long)sy * in_w + sx] : 0;
        v01 = (sx + 1 < in_w && sy >= 0) ? src[(long)sy * in_w + sx + 1] : 0;
        v10 = (sx >= 0 && sy + 1 < in_h) ? src[(long)(sy + 1) * in_w + sx] : 0;
        v11 = (sx + 1 < in_w && sy + 1 < in_h) ? src[(long)(sy + 1) * in_w + sx + 1] : 0;
        dst[p] = (uint8_t)((v00 * w00 + v01 * w01 + v10 * w10 + v11 * w11 + (1 << 14)) >> 15);
    }
}
