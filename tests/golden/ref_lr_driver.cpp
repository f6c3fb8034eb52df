// ref_lr_driver.cpp -- C-ABI over the reference's own lrCheck and fillInv (src/PP.cpp:17-143), and PP::processDM with
// its lines 405-406 restored.  TEST INFRASTRUCTURE, used only by make_golden_lr.py, which compiles it together with an
// unmodified src/PP.cpp of a reference checkout against oracle/shim with the flags of oracle/Makefile's _ref build.
#include "PP.h"

#include <cstring>
#include <string>

// external linkage in PP.cpp, no declaration in PP.h
void lrCheck(Mat& lDis, Mat& rDis, Mat& lValid, Mat& rValid);
void fillInv(Mat& lDis, Mat& rDis, Mat& lValid, Mat& rValid);

static Mat to_mat(const unsigned char* src, int W, int H)
{
    Mat m = Mat::zeros(H, W, CV_8UC1);
    for (int y = 0; y < H; ++y) memcpy(m.ptr<unsigned char>(y), src + (size_t)y * W, W);
    return m;
}

static void from_mat(const Mat& m, unsigned char* dst, int W, int H)
{
    for (int y = 0; y < H; ++y) memcpy(dst + (size_t)y * W, m.ptr<unsigned char>(y), W);
}

extern "C" {

// lrCheck then fillInv on u8 maps: masks and filled maps
int ref_lr_check_fill(const unsigned char* l, const unsigned char* r, int W, int H, unsigned char* lvalid,
                      unsigned char* rvalid, unsigned char* lfill, unsigned char* rfill)
{
    Mat lDis = to_mat(l, W, H), rDis = to_mat(r, W, H);
    Mat lValid = Mat::zeros(H, W, CV_8UC1), rValid = Mat::zeros(H, W, CV_8UC1);   // DispEst.cpp:48-49
    lrCheck(lDis, rDis, lValid, rValid);
    from_mat(lValid, lvalid, W, H);
    from_mat(rValid, rvalid, W, H);
    fillInv(lDis, rDis, lValid, rValid);
    from_mat(lDis, lfill, W, H);
    from_mat(rDis, rfill, W, H);
    return 0;
}

// PP::processDM (PP.cpp:402-425) with lines 405-406 restored and the filter's arguments exposed:
//   lrCheck; fillInv; img.convertTo(img8UC3, CV_8UC3, 255); JointWMF::filter(disp, img8UC3, r, sigma, 256, 256, iter, w)
int ref_process_dm_lr(const float* limg, const float* rimg, const unsigned char* l, const unsigned char* r, int W, int H,
                      int radius, float sigma, int iter, int weight, unsigned char* lout, unsigned char* rout)
{
    static const char* kNames[6] = {"exp", "iv1", "iv2", "cos", "jac", "off"};   // JointWMF.h:503-508
    if (weight < 0 || weight > 5) return 1;
    Mat lDis = to_mat(l, W, H), rDis = to_mat(r, W, H);
    Mat lValid = Mat::zeros(H, W, CV_8UC1), rValid = Mat::zeros(H, W, CV_8UC1);
    lrCheck(lDis, rDis, lValid, rValid);
    fillInv(lDis, rDis, lValid, rValid);
    Mat lImg(H, W, CV_32FC3, (void*)limg), rImg(H, W, CV_32FC3, (void*)rimg);
    Mat lImg8, rImg8;
    lImg.convertTo(lImg8, CV_8UC3, 255);
    rImg.convertTo(rImg8, CV_8UC3, 255);
    from_mat(JointWMF::filter(lDis, lImg8, radius, sigma, 256, 256, iter, std::string(kNames[weight])), lout, W, H);
    from_mat(JointWMF::filter(rDis, rImg8, radius, sigma, 256, 256, iter, std::string(kNames[weight])), rout, W, H);
    return 0;
}

}  // extern "C"
