// ref_wmf_driver.cpp -- C-ABI over the reference's own include/JointWMF.h at any (r, sigma, iter, weightType).
// TEST INFRASTRUCTURE, used only by make_golden_pp.py, which compiles it against a checkout of the reference
// (JointWMF.h unmodified) and oracle/shim with the flags of oracle/Makefile's _ref build.
// One view of PP::processDM's live code (src/PP.cpp:414-422) with the filter's arguments exposed:
//   img.convertTo(img8UC3, CV_8UC3, 255);  JointWMF::filter(disp, img8UC3, r, sigma, 256, 256, iter, weightType)
#include "JointWMF.h"

#include <vector>

extern "C" {

int ref_wmf(const float* img, const unsigned char* disp, int W, int H, int r, float sigma, int iter, int weight,
            unsigned char* out, int* n_colours)
{
    static const char* kNames[6] = {"exp", "iv1", "iv2", "cos", "jac", "off"};   // JointWMF.h:503-508
    if (weight < 0 || weight > 5) return 1;
    Mat Img(H, W, CV_32FC3, (void*)img);
    Mat Img8;
    Img.convertTo(Img8, CV_8UC3, 255);
    std::vector<unsigned char> seen(64 * 64 * 64, 0);   // distinct 6-bit colours (what JointWMF.h:552-568 counts)
    int cnt = 0;
    for (int y = 0; y < H; ++y) {
        const unsigned char* p = Img8.ptr<unsigned char>(y);
        for (int x = 0; x < W; ++x) {
            const int k = ((p[3 * x] >> 2) * 64 + (p[3 * x + 1] >> 2)) * 64 + (p[3 * x + 2] >> 2);
            if (!seen[k]) { seen[k] = 1; ++cnt; }
        }
    }
    *n_colours = cnt;
    Mat D = Mat::zeros(H, W, CV_8UC1);
    for (int y = 0; y < H; ++y) memcpy(D.ptr<unsigned char>(y), disp + (size_t)y * W, W);
    Mat res = JointWMF::filter(D, Img8, r, sigma, 256, 256, iter, std::string(kNames[weight]));
    for (int y = 0; y < H; ++y) memcpy(out + (size_t)y * W, res.ptr<unsigned char>(y), W);
    return 0;
}

}  // extern "C"
