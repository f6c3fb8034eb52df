// ref_wmf32f_driver.cpp -- C-ABI over the reference's own include/JointWMF.h with a CV_32F disparity map.
// TEST INFRASTRUCTURE, used only by make_golden_wide.py, which compiles it against a checkout of the reference
// (JointWMF.h unmodified) and oracle/shim with the flags of oracle/Makefile's _ref build.
// One view of PP::processDM's live code (src/PP.cpp:414-422) on a map wider than 8 bits:
//   img.convertTo(img8UC3, CV_8UC3, 255);  JointWMF::filter(disp as CV_32F, img8UC3, r, sigma, nI, 256, iter, weightType)
// For a map of integer values with at most nI distinct values from32FTo32S gives every value its own index and
// from32STo32F maps it back exactly, so this is the weighted median on the map's own values.
#include "JointWMF.h"

#include <vector>

extern "C" {

int ref_wmf32f(const float* img, const float* disp, int W, int H, int r, float sigma, int nI, int iter, int weight,
               float* out, int* n_colours)
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
    Mat D(H, W, CV_32FC1);
    for (int y = 0; y < H; ++y) memcpy(D.ptr<float>(y), disp + (size_t)y * W, (size_t)W * sizeof(float));
    Mat res = JointWMF::filter(D, Img8, r, sigma, nI, 256, iter, std::string(kNames[weight]));
    for (int y = 0; y < H; ++y) memcpy(out + (size_t)y * W, res.ptr<float>(y), (size_t)W * sizeof(float));
    return 0;
}

}  // extern "C"
