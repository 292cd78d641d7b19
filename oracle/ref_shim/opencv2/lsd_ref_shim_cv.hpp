// oracle/ref_shim/opencv2 -- TEST INFRASTRUCTURE, not product code and not OpenCV.
// The reference's hot-path sources use OpenCV only for debug images (cv::Mat members of DepthMap / SE3Tracker that are
// written under the plot* / debug flags of util/settings.cpp, all false by default) and for display.  This header gives
// those names a small self-contained implementation so that the reference files compile unmodified into oracle/_ref/;
// drawing and file output are no-ops.  Nothing here takes part in any number the oracle/_ref library returns, except the
// storage of util/Undistorter.cpp's UndistorterPTAM: the CV_64F K matrices it fills through at<double>() and the CV_8U image
// its undistort() writes through OutputArray, both plain element storage here.
#ifndef LSD_REF_SHIM_CV
#define LSD_REF_SHIM_CV
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <list>
#include <map>
#include <memory>
#include <string>
#include <vector>
#include <sys/time.h>
// opencv2/core/types_c.h (OpenCV 2.4) includes the C header <math.h>.  With g++ >= 6 that is libstdc++'s wrapper, which puts
// the float overloads of sqrt / abs / ... into the GLOBAL namespace, so the reference's unqualified `sqrt(float)` calls
// (DepthMap.cpp:229, 336, 1517, 1597) are float operations.  With the g++ 4.6 / 4.8 of the reference's own era
// (Ubuntu 12.04 / 14.04, README.md) the same calls resolve to `double sqrt(double)`; only DepthMap.cpp:229
// (`GRADIENT_SAMPLE_DIST / sqrt(eplLengthSquared)`, then evaluated in double) changes value, by <= 1 ulp.
// -DLSD_REF_SHIM_LEGACY_MATH builds that variant (tests/test_ref_pin.py measures its distance).  The same switch turns the
// unqualified tan / atan / sqrt of util/Undistorter.cpp into double operations (tests/test_ref_pin_undistort.py measures that).
#ifndef LSD_REF_SHIM_LEGACY_MATH
#include <math.h>
#endif

typedef unsigned char uchar;          /* opencv2/core/types_c.h puts these into the global namespace */
typedef unsigned short ushort;

#define CV_8U 0
#define CV_32F 5
#define CV_64F 6
#define CV_MAKETYPE(depth, cn) ((depth) + (((cn) - 1) << 3))
#define CV_8UC1 CV_MAKETYPE(CV_8U, 1)
#define CV_8UC3 CV_MAKETYPE(CV_8U, 3)
#define CV_8UC4 CV_MAKETYPE(CV_8U, 4)
#define CV_32FC1 CV_MAKETYPE(CV_32F, 1)
#define CV_32FC3 CV_MAKETYPE(CV_32F, 3)
#define CV_64FC1 CV_MAKETYPE(CV_64F, 1)
#define CV_GRAY2RGB 8
#define CV_GRAY2BGR 8
#define CV_RGB2GRAY 7
#define CV_BGR2GRAY 6
#define CV_AA 16
#define CV_FONT_HERSHEY_SIMPLEX 0

namespace cv {

template<typename T, int N> struct Vec {
    T val[N];
    Vec() { for (int i = 0; i < N; ++i) val[i] = T(); }
    Vec(T a, T b, T c) { static_assert(N == 3, "3 channels"); val[0] = a; val[1] = b; val[2] = c; }
    Vec(T a, T b, T c, T d) { static_assert(N == 4, "4 channels"); val[0] = a; val[1] = b; val[2] = c; val[3] = d; }
    T& operator[](int i) { return val[i]; }
    const T& operator[](int i) const { return val[i]; }
};
typedef Vec<unsigned char, 3> Vec3b;
typedef Vec<unsigned char, 4> Vec4b;
typedef Vec<float, 3> Vec3f;

struct Scalar {
    double val[4];
    Scalar(double a = 0, double b = 0, double c = 0, double d = 0) { val[0] = a; val[1] = b; val[2] = c; val[3] = d; }
    double& operator[](int i) { return val[i]; }
};
template<typename T> struct Point_ {
    T x, y;
    Point_() : x(0), y(0) {}
    Point_(T a, T b) : x(a), y(b) {}
};
typedef Point_<int> Point;
typedef Point_<float> Point2f;
typedef Point_<double> Point2d;
struct Size { int width, height; Size(int w = 0, int h = 0) : width(w), height(h) {} };

class Mat {
public:
    int rows, cols;
    unsigned char* data;
    Mat() : rows(0), cols(0), data(nullptr), type_(0), esz_(0) {}
    Mat(int r, int c, int type) { create(r, c, type); }
    Mat(int r, int c, int type, void* ext) : rows(r), cols(c), data(static_cast<unsigned char*>(ext)), type_(type), esz_(elem(type)) {}
    Mat(Size s, int type) { create(s.height, s.width, type); }
    Mat(int r, int c, int type, const Scalar& v)
    {
        create(r, c, type);
        for (int i = 0; i < r * c * channels(); ++i) setElem(i, v.val[0]);
    }
    static Mat zeros(int r, int c, int type) { return Mat(r, c, type); }
    bool isContinuous() const { return true; }
    // single-channel transpose (util/Undistorter.cpp:556-557)
    Mat t() const
    {
        Mat m(cols, rows, type_);
        for (int y = 0; y < rows; ++y)
            for (int x = 0; x < cols; ++x) std::memcpy(m.data + (static_cast<size_t>(x) * rows + y) * esz_, data + (static_cast<size_t>(y) * cols + x) * esz_, esz_);
        return m;
    }
    void create(int r, int c, int type)
    {
        rows = r; cols = c; type_ = type; esz_ = elem(type);
        own_.reset(new std::vector<unsigned char>(static_cast<size_t>(r) * c * esz_ + 16, 0));
        data = own_->data();
    }
    int type() const { return type_; }
    int channels() const { return (type_ >> 3) + 1; }
    bool empty() const { return data == nullptr || rows * cols == 0; }
    size_t elemSize() const { return esz_; }
    Size size() const { return Size(cols, rows); }
    template<typename T> T& at(int y, int x) { return *reinterpret_cast<T*>(data + (static_cast<size_t>(y) * cols + x) * esz_); }
    template<typename T> const T& at(int y, int x) const { return *reinterpret_cast<const T*>(data + (static_cast<size_t>(y) * cols + x) * esz_); }
    Mat clone() const { Mat m(rows, cols, type_); if (data) std::memcpy(m.data, data, static_cast<size_t>(rows) * cols * esz_); return m; }
    void copyTo(Mat& o) const { o = clone(); }
    void setTo(const Scalar&) {}
    void release() { own_.reset(); data = nullptr; rows = cols = 0; }
    // value conversion of debug images: geometry only (contents of debug plots are not part of any returned number)
    void convertTo(Mat& dst, int type, double = 1.0, double = 0.0) const { if (&dst != this) dst.create(rows, cols, type); }
private:
    void setElem(int i, double v)
    {
        switch (type_ & 7) {
        case CV_8U: data[i] = static_cast<unsigned char>(v); break;
        case CV_32F: reinterpret_cast<float*>(data)[i] = static_cast<float>(v); break;
        case CV_64F: reinterpret_cast<double*>(data)[i] = v; break;
        default: std::abort();
        }
    }
    static int elem(int type) { static const int dsz[8] = {1, 1, 2, 2, 4, 4, 8, 2}; return dsz[type & 7] * ((type >> 3) + 1); }
    int type_, esz_;
    std::shared_ptr<std::vector<unsigned char> > own_;
};
inline Mat operator*(double, const Mat& m) { return m; }
inline Mat operator*(const Mat& m, double) { return m; }
inline Mat operator+(const Mat& a, const Mat&) { return a; }
inline Mat operator-(const Mat& a, const Mat&) { return a; }

inline void cvtColor(const Mat& src, Mat& dst, int code, int = 0)
{
    const int r = src.rows, c = src.cols;
    if (code == CV_GRAY2RGB) dst.create(r, c, CV_8UC3);
    else dst.create(r, c, CV_8UC1);
}
inline void line(Mat&, Point2f, Point2f, const Scalar&, int = 1, int = 8, int = 0) {}
inline void circle(Mat&, Point, int, const Scalar&, int = 1, int = 8, int = 0) {}
inline void rectangle(Mat&, Point, Point, const Scalar&, int = 1, int = 8, int = 0) {}
inline void putText(Mat&, const std::string&, Point, int, double, const Scalar&, int = 1, int = 8, bool = false) {}
inline bool imwrite(const std::string&, const Mat&) { return false; }
inline Mat imread(const std::string&, int = 1) { return Mat(); }
inline void imshow(const std::string&, const Mat&) {}
inline int waitKey(int = 0) { return -1; }
inline void namedWindow(const std::string&, int = 0) {}
inline void destroyAllWindows() {}
inline void resize(const Mat& s, Mat& d, Size sz, double = 0, double = 0, int = 1) { d.create(sz.height, sz.width, s.type()); }

// the output-argument proxy of Undistorter::undistort (util/Undistorter.h:39): getMatRef() and create() of the wrapped Mat
class _OutputArray {
public:
    _OutputArray(Mat& m) : m_(&m) {}
    Mat& getMatRef() const { return *m_; }
    void create(int r, int c, int type) const { m_->create(r, c, type); }
private:
    Mat* m_;
};
typedef const _OutputArray& OutputArray;

// UndistorterOpenCV::undistort (Undistorter.cpp:564-567) is compiled but never run from oracle/_ref: reaching it is a bug
enum { INTER_LINEAR = 1 };
inline void remap(const Mat&, OutputArray, const Mat&, const Mat&, int, int = 0, const Scalar& = Scalar())
{
    std::fprintf(stderr, "oracle/ref_shim: cv::remap is not implemented (UndistorterOpenCV is not part of oracle/_ref)\n");
    std::abort();
}
}  // namespace cv
#endif
