/* Minimal stand-in for <opencv2/opencv.hpp> -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Purpose: let the UNMODIFIED reference sources (code/esac/esac.cpp, esac_util.h, esac_loss.h,
 * esac_derivative.h, thread_rand.cpp) compile in an image that has no OpenCV C++ headers or libraries, only the `cv2`
 * Python wheel (OpenCV 4.13, statically linked, no exported C++ symbols).  This header declares exactly the slice of
 * the cv:: API those files use.  The arithmetic that matters is NOT restated here:
 *   cv::solvePnP, cv::Rodrigues, cv::Mat::inv, cv::projectPoints  ->  executed by the real OpenCV inside the cv2 module
 *                                                                     (oracle/ref_shim/shim_cv2.cpp, via pybind11);
 *   element-wise ops, transposes, products of small double matrices, norms, traces -> plain IEEE double loops below.
 * Built by oracle/build_ref.py into oracle/_ref/.  Only tests/, bench.py's reference / cpu_baseline legs and
 * tests/golden/make_ref_golden.py use the result.
 */
#ifndef ESAC_REF_SHIM_OPENCV_HPP
#define ESAC_REF_SHIM_OPENCV_HPP

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <vector>

#define CV_8U 0
#define CV_32S 4
#define CV_32F 5
#define CV_64F 6
#define CV_PI 3.1415926535897932384626433832795

typedef unsigned char uchar; /* global, as in OpenCV's interface.h */

namespace cv {

using ::uchar;

enum { SOLVEPNP_ITERATIVE = 0, SOLVEPNP_EPNP = 1, SOLVEPNP_P3P = 2 };
enum { DECOMP_LU = 0, DECOMP_SVD = 1 };

template <typename T> struct Point_ {
    T x, y;
    Point_() : x(0), y(0) {}
    Point_(T x_, T y_) : x(x_), y(y_) {}
    template <typename U> Point_(const Point_<U>& o) : x((T)o.x), y((T)o.y) {}
};
template <typename T> inline Point_<T> operator-(const Point_<T>& a, const Point_<T>& b) { return Point_<T>((T)(a.x - b.x), (T)(a.y - b.y)); }
template <typename T> inline Point_<T> operator+(const Point_<T>& a, const Point_<T>& b) { return Point_<T>((T)(a.x + b.x), (T)(a.y + b.y)); }
template <typename T> inline double norm(const Point_<T>& p) { return std::sqrt((double)p.x * p.x + (double)p.y * p.y); }
typedef Point_<int> Point2i;
typedef Point_<float> Point2f;
typedef Point_<double> Point2d;

template <typename T> struct Point3_ {
    T x, y, z;
    Point3_() : x(0), y(0), z(0) {}
    Point3_(T x_, T y_, T z_) : x(x_), y(y_), z(z_) {}
};
typedef Point3_<float> Point3f;

struct Size {
    int width, height;
    Size() : width(0), height(0) {}
    Size(int w, int h) : width(w), height(h) {}
};

struct Scalar {
    double val[4];
    Scalar(double a = 0, double b = 0, double c = 0, double d = 0) { val[0] = a; val[1] = b; val[2] = c; val[3] = d; }
    double operator[](int i) const { return val[i]; }
};

template <typename T> struct DepthOf;
template <> struct DepthOf<uchar> { enum { type = CV_8U, channels = 1 }; };
template <> struct DepthOf<int> { enum { type = CV_32S, channels = 1 }; };
template <> struct DepthOf<float> { enum { type = CV_32F, channels = 1 }; };
template <> struct DepthOf<double> { enum { type = CV_64F, channels = 1 }; };
template <> struct DepthOf<Point2i> { enum { type = CV_32S + 8, channels = 2 }; };  /* CV_32SC2 */

/* Reference-counted dense 2-D matrix; row/col ranges are views into the same storage (like cv::Mat). */
class Mat {
public:
    int rows, cols;
    Mat() : rows(0), cols(0), type_(0), esz_(1), step_(0), data_(nullptr) {}
    Mat(int r, int c, int type) { create(r, c, type); }
    Mat(const Point3f& p) { create(3, 1, CV_32F); at<float>(0, 0) = p.x; at<float>(1, 0) = p.y; at<float>(2, 0) = p.z; }

    void create(int r, int c, int type) {
        rows = r; cols = c; type_ = type;
        esz_ = elem_size(type);
        step_ = (size_t)c * esz_;
        buf_ = std::make_shared<std::vector<unsigned char>>((size_t)r * step_ + 16, (unsigned char)0);
        data_ = buf_->data();
    }
    static size_t elem_size(int type) {
        switch (type) {
            case CV_8U: return 1;
            case CV_32S: return 4;
            case CV_32F: return 4;
            case CV_64F: return 8;
            case CV_32S + 8: return 8;
            default: throw std::runtime_error("shim cv::Mat: unsupported type");
        }
    }
    int type() const { return type_; }
    int depth() const { return type_ & 7; }
    bool empty() const { return rows == 0 || cols == 0 || data_ == nullptr; }
    Size size() const { return Size(cols, rows); }
    size_t step() const { return step_; }
    bool isContinuous() const { return step_ == (size_t)cols * esz_ || rows <= 1; }
    unsigned char* ptr(int r = 0) { return data_ + (size_t)r * step_; }
    const unsigned char* ptr(int r = 0) const { return data_ + (size_t)r * step_; }

    template <typename T> T& at(int r, int c) { return *reinterpret_cast<T*>(data_ + (size_t)r * step_ + (size_t)c * esz_); }
    template <typename T> const T& at(int r, int c) const { return *reinterpret_cast<const T*>(data_ + (size_t)r * step_ + (size_t)c * esz_); }
    /* single index: element i of a 1 x n or n x 1 matrix (cv::Mat::at(int i0)) */
    template <typename T> T& at(int i) { return rows == 1 ? at<T>(0, i) : at<T>(i, 0); }
    template <typename T> const T& at(int i) const { return rows == 1 ? at<T>(0, i) : at<T>(i, 0); }

    Mat rowRange(int a, int b) const { Mat m(*this); m.data_ = data_ + (size_t)a * step_; m.rows = b - a; return m; }
    Mat colRange(int a, int b) const { Mat m(*this); m.data_ = data_ + (size_t)a * esz_; m.cols = b - a; return m; }
    Mat row(int i) const { return rowRange(i, i + 1); }
    Mat col(int i) const { return colRange(i, i + 1); }

    Mat clone() const {
        Mat m;
        if (data_ == nullptr) { m.type_ = type_; return m; }
        m.create(rows, cols, type_);
        for (int r = 0; r < rows; r++) std::memcpy(m.ptr(r), ptr(r), (size_t)cols * esz_);
        return m;
    }
    /* copyTo an lvalue (re-allocated when the shape differs) or into a view (shape must match) */
    void copyTo(Mat& dst) const {
        if (dst.rows != rows || dst.cols != cols || dst.type_ != type_ || dst.data_ == nullptr) dst.create(rows, cols, type_);
        for (int r = 0; r < rows; r++) std::memmove(dst.ptr(r), ptr(r), (size_t)cols * esz_);
    }
    void copyTo(Mat&& view) const {
        if (view.rows != rows || view.cols != cols || view.type_ != type_) throw std::runtime_error("shim cv::Mat::copyTo: view shape/type mismatch");
        for (int r = 0; r < rows; r++) std::memmove(view.ptr(r), ptr(r), (size_t)cols * esz_);
    }
    void convertTo(Mat& dst, int type) const;

    double get(int r, int c) const {
        switch (type_) {
            case CV_8U: return at<uchar>(r, c);
            case CV_32S: return at<int>(r, c);
            case CV_32F: return at<float>(r, c);
            case CV_64F: return at<double>(r, c);
            default: throw std::runtime_error("shim cv::Mat::get: unsupported type");
        }
    }
    void set(int r, int c, double v) {
        switch (type_) {
            case CV_8U: at<uchar>(r, c) = (uchar)v; break;
            case CV_32S: at<int>(r, c) = (int)std::lrint(v); break;
            case CV_32F: at<float>(r, c) = (float)v; break;
            case CV_64F: at<double>(r, c) = v; break;
            default: throw std::runtime_error("shim cv::Mat::set: unsupported type");
        }
    }

    Mat t() const;
    Mat inv(int method = DECOMP_LU) const; /* real OpenCV: cv2.invert */

    Mat& operator+=(const Mat& b);
    Mat& operator-=(const Mat& b);
    Mat& operator*=(double s);
    void setTo(double v) { for (int r = 0; r < rows; r++) for (int c = 0; c < cols; c++) set(r, c, v); }

protected:
    int type_;
    size_t esz_, step_;
    unsigned char* data_;
    std::shared_ptr<std::vector<unsigned char>> buf_;
};

inline void Mat::convertTo(Mat& dst, int type) const {
    Mat out(rows, cols, type);
    for (int r = 0; r < rows; r++) for (int c = 0; c < cols; c++) out.set(r, c, get(r, c));
    dst = out;
}

template <typename T> class Mat_ : public Mat {
public:
    Mat_() : Mat() { type_ = DepthOf<T>::type; esz_ = sizeof(T); }
    Mat_(int r, int c) : Mat(r, c, DepthOf<T>::type) {}
    explicit Mat_(Size s) : Mat(s.height, s.width, DepthOf<T>::type) {}
    Mat_(const Mat& m) : Mat() { assign(m); }
    Mat_(const Mat_& m) : Mat(static_cast<const Mat&>(m)) {}
    Mat_& operator=(const Mat& m) { assign(m); return *this; }
    Mat_& operator=(const Mat_& m) { Mat::operator=(static_cast<const Mat&>(m)); return *this; }
    Mat_& operator=(const T& v) { for (int r = 0; r < rows; r++) for (int c = 0; c < cols; c++) (*this)(r, c) = v; return *this; }

    T& operator()(int r, int c) { return this->template at<T>(r, c); }
    const T& operator()(int r, int c) const { return this->template at<T>(r, c); }
    T& operator()(int i) { return this->template at<T>(i); }
    const T& operator()(int i) const { return this->template at<T>(i); }

    Mat_ clone() const { return Mat_(Mat::clone()); }

    static Mat_ zeros(int r, int c) { return Mat_(r, c); }
    static Mat_ zeros(Size s) { return Mat_(s); }
    static Mat_ eye(int r, int c) { Mat_ m(r, c); for (int i = 0; i < std::min(r, c); i++) m(i, i) = (T)1; return m; }

private:
    void assign(const Mat& m) {
        if (m.type() == (int)DepthOf<T>::type || m.rows == 0 || m.cols == 0) {
            Mat::operator=(m);
            if (m.rows == 0 || m.cols == 0) { type_ = DepthOf<T>::type; esz_ = sizeof(T); }
        } else {
            Mat tmp;
            m.convertTo(tmp, DepthOf<T>::type);
            Mat::operator=(tmp);
        }
    }
};

/* ---- arithmetic on double / float matrices (results are CV_64F unless both operands are CV_32F) ---- */
Mat operator*(const Mat& a, const Mat& b);
Mat operator+(const Mat& a, const Mat& b);
Mat operator-(const Mat& a, const Mat& b);
Mat operator-(const Mat& a);
Mat operator*(const Mat& a, double s);
Mat operator*(double s, const Mat& a);
Mat operator/(const Mat& a, double s);
Mat operator!=(const Mat& a, const Mat& b); /* CV_8U mask, 255 where different (NaN != NaN) */

Scalar trace(const Mat& m);
Scalar sum(const Mat& m);
double norm(const Mat& m); /* L2 */

/* ---- calib3d: executed by the real OpenCV through the cv2 module (shim_cv2.cpp) ---- */
bool solvePnP(const std::vector<Point3f>& objectPoints, const std::vector<Point2f>& imagePoints, const Mat& cameraMatrix,
              const Mat& distCoeffs, Mat& rvec, Mat& tvec, bool useExtrinsicGuess = false, int flags = SOLVEPNP_ITERATIVE);
void projectPoints(const std::vector<Point3f>& objectPoints, const Mat& rvec, const Mat& tvec, const Mat& cameraMatrix,
                   const Mat& distCoeffs, std::vector<Point2f>& imagePoints);
void projectPoints(const std::vector<Point3f>& objectPoints, const Mat& rvec, const Mat& tvec, const Mat& cameraMatrix,
                   const Mat& distCoeffs, std::vector<Point2f>& imagePoints, Mat& jacobian);
void Rodrigues(const Mat& src, Mat& dst);
void Rodrigues(const Mat& src, Mat& dst, Mat& jacobian);

}  // namespace cv

#endif
