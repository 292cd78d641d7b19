// oracle/ref_shim/opencv2/calib3d -- TEST INFRASTRUCTURE, not OpenCV.  Declarations util/Undistorter.cpp needs to compile.
// Only UndistorterOpenCV's constructor (Undistorter.cpp:545-548) calls these; oracle/_ref never constructs that class (it is
// pinned to OpenCV itself by tests/golden/opencv_undistort.npz), so reaching either one aborts.
#ifndef LSD_REF_SHIM_CV_CALIB3D
#define LSD_REF_SHIM_CV_CALIB3D
#include "../lsd_ref_shim_cv.hpp"

#define CV_16SC2 CV_MAKETYPE(3, 2)

namespace cv {
struct Rect;
inline void lsd_ref_shim_unimplemented(const char* what)
{
    std::fprintf(stderr, "oracle/ref_shim: cv::%s is not implemented (UndistorterOpenCV is not part of oracle/_ref)\n", what);
    std::abort();
}
inline Mat getOptimalNewCameraMatrix(const Mat&, const Mat&, Size, double, Size = Size(), Rect* = nullptr, bool = false)
{
    lsd_ref_shim_unimplemented("getOptimalNewCameraMatrix");
    return Mat();
}
inline void initUndistortRectifyMap(const Mat&, const Mat&, const Mat&, const Mat&, Size, int, Mat&, Mat&)
{
    lsd_ref_shim_unimplemented("initUndistortRectifyMap");
}
}  // namespace cv
#endif
