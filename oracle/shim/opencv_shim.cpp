// opencv_shim.cpp -- the six image primitives behind oracle/shim/opencv2/opencv.hpp.
// TEST INFRASTRUCTURE ONLY (part of oracle/_ref).  Each primitive forwards to the C restatement in
// oracle/stereo_oracle.c, which is pinned against python cv2 (tests/test_oracle.py).
#include <opencv2/opencv.hpp>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../stereo_oracle.h"

namespace {
int g_gray_mode = 0;

void need(bool ok, const char* what)
{
    if (!ok) { std::fprintf(stderr, "opencv shim: unsupported use: %s\n", what); std::abort(); }
}

// contiguous copy of a 1-channel float Mat (the C primitives take packed planes)
std::vector<float> packed(const cv::Mat& m)
{
    const int cn = m.channels();
    std::vector<float> v((size_t)m.rows * m.cols * cn);
    for (int y = 0; y < m.rows; ++y) std::memcpy(&v[(size_t)y * m.cols * cn], m.ptr<float>(y), (size_t)m.cols * cn * sizeof(float));
    return v;
}
void unpack(const std::vector<float>& v, cv::Mat& dst, int rows, int cols)
{
    dst.create(rows, cols, CV_32FC1);
    for (int y = 0; y < rows; ++y) std::memcpy(dst.ptr<float>(y), &v[(size_t)y * cols], (size_t)cols * sizeof(float));
}
}  // namespace

extern "C" void psm_shim_set_gray_mode(int mode) { g_gray_mode = mode; }

namespace cv {

Mat& Mat::operator-=(const Mat& o)
{
    need(type() == CV_32FC1 && o.type() == CV_32FC1 && rows == o.rows && cols == o.cols, "Mat -= Mat (CV_32FC1, same size)");
    for (int y = 0; y < rows; ++y) {
        float* a = ptr<float>(y);
        const float* b = o.ptr<float>(y);
        for (int x = 0; x < cols; ++x) a[x] = a[x] - b[x];
    }
    return *this;
}

Mat& Mat::operator+=(const Mat& o)
{
    need(type() == CV_32FC1 && o.type() == CV_32FC1 && rows == o.rows && cols == o.cols, "Mat += Mat (CV_32FC1, same size)");
    for (int y = 0; y < rows; ++y) {
        float* a = ptr<float>(y);
        const float* b = o.ptr<float>(y);
        for (int x = 0; x < cols; ++x) a[x] = a[x] + b[x];
    }
    return *this;
}

Mat operator-(const Mat& a, const Mat& b)
{
    need(a.type() == CV_32FC1 && b.type() == CV_32FC1 && a.rows == b.rows && a.cols == b.cols, "Mat - Mat (CV_32FC1, same size)");
    Mat r(a.rows, a.cols, CV_32FC1);
    for (int y = 0; y < a.rows; ++y) {
        const float* pa = a.ptr<float>(y);
        const float* pb = b.ptr<float>(y);
        float* pr = r.ptr<float>(y);
        for (int x = 0; x < a.cols; ++x) pr[x] = pa[x] - pb[x];
    }
    return r;
}

Mat& Mat::operator=(const Scalar& sc)
{
    need(channels() == 1, "Mat = Scalar on a 1-channel Mat");
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            if (depth() == CV_8U) at<uchar>(y, x) = (uchar)sc.val[0];
            else if (depth() == CV_32S) at<int>(y, x) = (int)sc.val[0];
            else at<float>(y, x) = (float)sc.val[0];
        }
    return *this;
}

void Mat::convertTo(Mat& dst, int rtype, double alpha, double beta) const
{
    const int cn = channels(), sd = depth(), dd = CV_MAT_DEPTH(rtype);
    Mat out(rows, cols, CV_MAKETYPE(dd, cn));
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols * cn; ++x) {
            if (sd == CV_8U && dd == CV_32S) { need(alpha == 1.0 && beta == 0.0, "convertTo scale"); out.ptr<int>(y)[x] = ptr<uchar>(y)[x]; }
            else if (sd == CV_32S && dd == CV_8U) { need(alpha == 1.0 && beta == 0.0, "convertTo scale"); int v = ptr<int>(y)[x]; out.ptr<uchar>(y)[x] = (uchar)(v < 0 ? 0 : (v > 255 ? 255 : v)); }
            else if (sd == CV_32F && dd == CV_8U) {  // cv::saturate_cast<uchar>(cvRound(v*alpha)): the C restatement
                need(alpha == 255.0 && beta == 0.0, "convertTo 32F -> 8U scale other than 255");
                orc_f32_to_u8x255(ptr<float>(y) + x, out.ptr<uchar>(y) + x, 1);
            } else need(false, "convertTo: unsupported depth pair");
        }
    dst = out;
}

void split(const Mat& src, std::vector<Mat>& mv)
{
    need(src.channels() == 1, "split(vector) of a 1-channel Mat");
    mv.assign(1, src.clone());
}

void merge(const std::vector<Mat>& mv, Mat& dst)
{
    need(mv.size() == 1, "merge of one channel");
    dst = mv[0].clone();
}

void minMaxLoc(const Mat& src, double* minVal, double* maxVal)
{
    need(src.type() == CV_32FC1, "minMaxLoc(CV_32FC1)");
    double lo = DBL_MAX, hi = -DBL_MAX;
    for (int y = 0; y < src.rows; ++y)
        for (int x = 0; x < src.cols; ++x) { const double v = src.at<float>(y, x); lo = v < lo ? v : lo; hi = v > hi ? v : hi; }
    if (minVal) *minVal = lo;
    if (maxVal) *maxVal = hi;
}

double kmeans(const Mat& samples, int K, Mat& labels, TermCriteria, int, int, Mat& centers)
{
    need(samples.type() == CV_32FC1 && samples.cols == 3 && K >= 1 && K <= samples.rows, "kmeans(N x 3 CV_32F)");
    const int N = samples.rows;
    labels.create(N, 1, CV_32SC1);
    centers.create(K, 3, CV_32FC1);
    if (K == N) {   // every sample is its own centre: exact, order-independent
        for (int i = 0; i < N; ++i) { labels.at<int>(i, 0) = i; std::memcpy(centers.ptr<float>(i), samples.ptr<float>(i), 12); }
        return 0.0;
    }
    // deterministic stand-in (NOT cv::kmeans): farthest-point seeding from sample 0, then two Lloyd iterations
    std::vector<float> best(N, 3.4e38f);
    int pick = 0;
    for (int k = 0; k < K; ++k) {
        std::memcpy(centers.ptr<float>(k), samples.ptr<float>(pick), 12);
        float far = -1.f; int arg = 0;
        for (int i = 0; i < N; ++i) {
            const float* sp = samples.ptr<float>(i); const float* c = centers.ptr<float>(k);
            const float d = (sp[0]-c[0])*(sp[0]-c[0]) + (sp[1]-c[1])*(sp[1]-c[1]) + (sp[2]-c[2])*(sp[2]-c[2]);
            if (d < best[i]) best[i] = d;
            if (best[i] > far) { far = best[i]; arg = i; }
        }
        pick = arg;
    }
    for (int it = 0; it < 2; ++it) {
        std::vector<double> acc((size_t)K * 3, 0.0); std::vector<int> cnt(K, 0);
        for (int i = 0; i < N; ++i) {
            const float* sp = samples.ptr<float>(i); float bd = 3.4e38f; int bk = 0;
            for (int k = 0; k < K; ++k) {
                const float* c = centers.ptr<float>(k);
                const float d = (sp[0]-c[0])*(sp[0]-c[0]) + (sp[1]-c[1])*(sp[1]-c[1]) + (sp[2]-c[2])*(sp[2]-c[2]);
                if (d < bd) { bd = d; bk = k; }
            }
            labels.at<int>(i, 0) = bk; cnt[bk]++;
            for (int c3 = 0; c3 < 3; ++c3) acc[(size_t)bk * 3 + c3] += sp[c3];
        }
        if (it == 0)
            for (int k = 0; k < K; ++k) if (cnt[k]) for (int c3 = 0; c3 < 3; ++c3) centers.at<float>(k, c3) = (float)(acc[(size_t)k * 3 + c3] / cnt[k]);
    }
    return 0.0;
}

void split(const Mat& src, Mat* mv)
{
    need(src.type() == CV_32FC3, "split(CV_32FC3)");
    for (int c = 0; c < 3; ++c) mv[c].create(src.rows, src.cols, CV_32FC1);
    for (int y = 0; y < src.rows; ++y) {
        const float* s = src.ptr<float>(y);
        for (int c = 0; c < 3; ++c) {
            float* d = mv[c].ptr<float>(y);
            for (int x = 0; x < src.cols; ++x) d[x] = s[3 * x + c];
        }
    }
}

void boxFilter(const Mat& src, Mat& dst, int ddepth, Size ksize)
{
    need(src.type() == CV_32FC1 && ddepth == -1 && ksize.width == ORC_GIF_R_WIN && ksize.height == ORC_GIF_R_WIN,
         "boxFilter(CV_32FC1, -1, Size(8,8))");
    const int rows = src.rows, cols = src.cols;
    if (src.step == (size_t)cols * sizeof(float)) {   // packed rows: filter straight into the destination (orc_box allows src == dst)
        const Mat keep = src;                          // dst may be the same header as src
        dst.create(rows, cols, CV_32FC1);
        orc_box(keep.ptr<float>(0), cols, rows, ksize.width, dst.ptr<float>(0));
        return;
    }
    std::vector<float> in = packed(src), out(in.size());
    orc_box(in.data(), cols, rows, ksize.width, out.data());
    unpack(out, dst, rows, cols);
}

void multiply(const Mat& a, const Mat& b, Mat& dst, double scale, int dtype)
{
    need(a.type() == CV_32FC1 && b.type() == CV_32FC1 && a.rows == b.rows && a.cols == b.cols && scale == 1.0 && dtype == -1,
         "multiply(CV_32FC1, CV_32FC1)");
    const int rows = a.rows, cols = a.cols;
    Mat out = (dst.data == a.data || dst.data == b.data) ? dst : Mat();   // in-place use is legal (CVF.cpp:161)
    out.create(rows, cols, CV_32FC1);
    for (int y = 0; y < rows; ++y) {
        const float* pa = a.ptr<float>(y);
        const float* pb = b.ptr<float>(y);
        float* pd = out.ptr<float>(y);
        for (int x = 0; x < cols; ++x) pd[x] = pa[x] * pb[x];
    }
    dst = out;
}

void cvtColor(const Mat& src, Mat& dst, int code, int)
{
    need(src.type() == CV_32FC3 && code == CV_RGB2GRAY, "cvtColor(CV_32FC3, CV_RGB2GRAY)");
    std::vector<float> in = packed(src), out((size_t)src.rows * src.cols);
    orc_rgb2gray(in.data(), src.cols, src.rows, out.data(), g_gray_mode);
    unpack(out, dst, src.rows, src.cols);
}

void Sobel(const Mat& src, Mat& dst, int ddepth, int dx, int dy, int ksize)
{
    need(src.type() == CV_32FC1 && ddepth == CV_32F && dx == 1 && dy == 0 && ksize == 1, "Sobel(CV_32F, 1, 0, 1)");
    std::vector<float> in = packed(src), out(in.size());
    orc_sobel_x(in.data(), src.cols, src.rows, out.data());
    unpack(out, dst, src.rows, src.cols);
}

}  // namespace cv
