// DispEstB200.h -- C++ host facade with the reference's DispEst API surface
// (reference include/DispEst.h:21-109) whose "_GPU" stage methods run on the H100 C-ABI
// library (include/prime_stereo_b200.h) instead of the reference's OpenCL classes.
//
// Two ways to use it (INTEGRATION.md):
//   1. in the reference application: keep the reference's own DispEst.h/.cpp for the CPU stages and
//      patch the three _GPU bodies + ctor/dtor with the calls shown in INTEGRATION.md;
//   2. standalone (this header): compiles against OpenCV when its headers are present, otherwise
//      against the minimal cv::Mat stand-in below (this image has no OpenCV C++ headers).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>

#include "../../include/prime_stereo_b200.h"

#if !defined(PSM_NO_OPENCV) && defined(__has_include)
#if __has_include(<opencv2/core.hpp>)
#include <opencv2/core.hpp>
#define PSM_HAVE_OPENCV 1
#endif
#endif

#ifndef PSM_HAVE_OPENCV
// Minimal stand-in for the handful of cv::Mat members the facade touches.
#define CV_8U 0
#define CV_16U 2
#define CV_16S 3
#define CV_32F 5
#define CV_MAT_DEPTH_MASK 7
#define CV_MAKETYPE(depth, cn) ((depth) + (((cn)-1) << 3))
#define CV_8UC1 CV_MAKETYPE(CV_8U, 1)
#define CV_8UC2 CV_MAKETYPE(CV_8U, 2)
#define CV_8UC3 CV_MAKETYPE(CV_8U, 3)
#define CV_16UC1 CV_MAKETYPE(CV_16U, 1)
#define CV_16SC2 CV_MAKETYPE(CV_16S, 2)
#define CV_32FC1 CV_MAKETYPE(CV_32F, 1)
#define CV_32FC3 CV_MAKETYPE(CV_32F, 3)
namespace cv {
class Mat {
public:
    int rows = 0, cols = 0;
    size_t step = 0;
    unsigned char* data = nullptr;
    Mat() = default;
    Mat(int r, int c, int type) { create(r, c, type); }
    Mat(int r, int c, int type, void* ext, size_t ext_step) : rows(r), cols(c), step(ext_step), data((unsigned char*)ext), type_(type) {}
    static Mat zeros(int r, int c, int type) { Mat m(r, c, type); std::memset(m.data, 0, m.step * r); return m; }
    void create(int r, int c, int type)
    {
        rows = r; cols = c; type_ = type;
        step = (size_t)c * elemSize();
        owner_.reset(new unsigned char[step * r], std::default_delete<unsigned char[]>());
        data = owner_.get();
    }
    int type() const { return type_; }
    int channels() const { return (type_ >> 3) + 1; }
    size_t elemSize() const { return (size_t)channels() * ((type_ & CV_MAT_DEPTH_MASK) == CV_32F ? 4 : (type_ & CV_MAT_DEPTH_MASK) == CV_16U || (type_ & CV_MAT_DEPTH_MASK) == CV_16S ? 2 : 1); }
    bool empty() const { return data == nullptr; }
    template <typename T> T* ptr(int y = 0) { return (T*)(data + step * y); }
    template <typename T> const T* ptr(int y = 0) const { return (const T*)(data + step * y); }
private:
    int type_ = 0;
    std::shared_ptr<unsigned char> owner_;
};
}  // namespace cv
#endif

#define MAX_CPU_THREADS 8  // reference include/ComFunc.h:52
#define OCV_DE 0
#define OCL_DE 1

// Role of openCLdevicepoll() (reference src/main.cpp:29): number of compute devices; 0 disables the `m` toggle.
inline int b200devicepoll() { return psm_device_count(); }

class DispEst {
public:
    // reference src/DispEst.cpp:10-143.  `ocl` == use the GPU path.  block_slices > 0: a blocked context
    // (psm_create_blocked) that holds that many disparity slices at a time, for ranges the device cannot hold whole.
    // devices: empty = device 0; one id = that device; two or more = a multi-device context (psm_create_multi) whose
    // shard k runs on devices[k] (ids may repeat), each shard blocked by block_slices when it is > 0.  min_disp > 0: the
    // same kind of context over disparities [min_disp, d) alone (psm_create_range); the maps hold absolute disparities.
    DispEst(cv::Mat l, cv::Mat r, const int d, int t, bool ocl, int block_slices = 0, std::vector<int> devices = {},
            int min_disp = 0);
    ~DispEst(void);

    cv::Mat lDisMap;  // CV_8UC1, raw disparity index (reference DispEst.h:28-29); CV_16UC1 when maxDis > 256 (psm_create_u16),
                      // whose low byte is the reference's uchar map
    cv::Mat rDisMap;
    cv::Mat lValid;   // CV_8UC1 masks of the left-right check (reference DispEst.h:81-82), 0/1; PostProcess_GPU fills them
    cv::Mat rValid;   // when setLRCheck selected a mode other than PSM_LR_OFF (and no step of the chain an _ONLY mode);
                      // lValid alone on a left-only context that fills after setDisparityCheck(PSM_DCHECK_FIRST) or
                      // setUniquenessCheck(PSM_UNIQUE_FIRST)
    cv::Mat lCosts[3];  // setCostOutput(true): CV_32FC1 filtered costs at disparity m - 1, m, m + 1 of the selection map's
    cv::Mat rCosts[3];  // m (psm_read_costs); DispSelect_GPU fills them, rCosts not on a left-only context
    cv::Mat lRunnerUp[2];  // setRunnerUpOutput(true): CV_32FC1 runner-up disparity r (0 where none exists) and its
    cv::Mat rRunnerUp[2];  // filtered cost (psm_read_runner_up); DispSelect_GPU fills them, rRunnerUp not when left-only

    int setInputImages(cv::Mat l, cv::Mat r);
    // YUV frames as input (psm_set_images_yuv): format PSM_YUV_NV12 ... PSM_YUV_YVYU, frames in cv2's layouts -- CV_8UC1
    // of (H * 3 / 2) x W for the 4:2:0 formats, CV_8UC2 of H x W for the 4:2:2 ones, of the context's size or setRectify's
    // source size.  CostConst_GPU converts them to BGR on the device as cvtColor(COLOR_YUV2BGR_*) does.
    int setInputImagesYUV(cv::Mat l, cv::Mat r, int format);
    // Bayer raw frames as input (psm_set_images_bayer): pattern PSM_BAYER_RGGB ... PSM_BAYER_GBRG (the colours of the
    // 2 x 2 cell at (0, 0)), method PSM_DEMOSAIC_BILINEAR or PSM_DEMOSAIC_EA, CV_8UC1 frames of the context's size or
    // setRectify's source size.  CostConst_GPU demosaics them on the device as cvtColor(COLOR_Bayer*2BGR[_EA]) does.
    int setInputImagesBayer(cv::Mat l, cv::Mat r, int pattern, int method = PSM_DEMOSAIC_BILINEAR);
    int setThreads(unsigned int newThreads);
    void setSubsampleRate(unsigned int newRate) { subsample_rate = newRate; }
    // guided-filter window and eps (the reference's GIF_R_WIN / GIF_EPS) for the later CostFilter calls; see
    // psm_set_guided_filter.  INTEGRATION.md: call setGuidedFilter(GIF_R_WIN, GIF_EPS) so the GPU mode follows the build.
    int setGuidedFilter(int window, float eps);
    // matching-cost alpha and truncation thresholds (the reference's ALPHA_32F / TAU_1_32F / TAU_2_32F) for the later
    // CostConst calls; see psm_set_matching_cost.  INTEGRATION.md: setMatchingCost(ALPHA_32F, INFINITY, INFINITY).
    int setMatchingCost(float alpha, float tau_color, float tau_grad);
    // Weighted-median post-filter (JointWMF::filter's r, sigma, iter, weightType: PSM_WMF_*) for every later PostProcess
    // call; see psm_set_post_filter.  INTEGRATION.md: setPostFilter(MED_SZ/2, 25.5f, 1, PSM_WMF_EXP).
    int setPostFilter(int radius, float sigma, int iterations, int weight_type);
    // Left-right consistency check and occlusion fill in front of (PSM_LR_FILL_WMF) or instead of (PSM_LR_FILL) the
    // post-filter for every later PostProcess call; see psm_set_lr_check.  INTEGRATION.md: a build that restores
    // PP.cpp:405-406 calls setLRCheck(PSM_LR_FILL_WMF).
    int setLRCheck(int mode);
    // Speckle removal (cv::filterSpeckles(map, 0, max_size, max_diff)) in front of (PSM_SPECKLE_FIRST) or instead of
    // (PSM_SPECKLE_ONLY) the check and post-filter for every later PostProcess call; see psm_set_speckle_filter.  A port
    // of a StereoSGBM pipeline calls setSpeckleFilter(PSM_SPECKLE_FIRST, speckleWindowSize, speckleRange).
    int setSpeckleFilter(int mode, int max_size, int max_diff);
    // One-view disparity check (cv::validateDisparity, StereoSGBM's disp12MaxDiff) in front of (PSM_DCHECK_FIRST) or
    // instead of (PSM_DCHECK_ONLY) the speckle removal, check and post-filter for every later PostProcess call; see
    // psm_set_disparity_check.  It reads the winners' costs: call setCostOutput(true) before DispSelect_GPU.  A port of a
    // StereoSGBM pipeline calls setDisparityCheck(PSM_DCHECK_FIRST, disp12MaxDiff).
    int setDisparityCheck(int mode, int max_diff);
    // Uniqueness test (StereoSGBM's uniquenessRatio) at the head of (PSM_UNIQUE_FIRST) or instead of (PSM_UNIQUE_ONLY)
    // the rest of the post-process chain for every later PostProcess call; see psm_set_uniqueness_check.  It reads the
    // winners' costs and the runner-up: call setCostOutput(true) and setRunnerUpOutput(true) before DispSelect_GPU.  A
    // port of a StereoSGBM pipeline calls setUniquenessCheck(PSM_UNIQUE_FIRST, uniquenessRatio).
    int setUniquenessCheck(int mode, int ratio);
    // ksize x ksize median (cv::medianBlur; StereoSGBM::compute's fixed medianBlur(disp, 3)) after the uniqueness test and
    // disparity check, in front of (PSM_MEDIAN_FIRST) or instead of (PSM_MEDIAN_ONLY) the speckle removal, check and
    // post-filter for every later PostProcess call; see psm_set_median_blur.
    int setMedianBlur(int mode, int ksize);
    // PSM_VIEWS_BOTH (default) or PSM_VIEWS_LEFT (PSM_OPT_VIEWS): with PSM_VIEWS_LEFT the later frames compute the left
    // map alone; DispSelect_GPU and PostProcess_GPU then leave rDisMap (and rValid) untouched.  The next stage after a
    // change must be CostConst_GPU.
    int setViews(int views);
    // PSM_OPT_COSTS: with true, DispSelect_GPU also fills lCosts / rCosts.  The next stage after a change must be
    // CostConst_GPU.  Fails on a context that owns part of the disparity range.
    int setCostOutput(bool on);
    // PSM_OPT_RUNNER_UP: with true, DispSelect_GPU also fills lRunnerUp / rRunnerUp.  The next stage after a change must
    // be CostConst_GPU.  Fails on a context that owns part of the disparity range.
    int setRunnerUpOutput(bool on);
    // Rectify every later frame on the device (psm_set_rectify): the reference's video-mode remap(frame, rec, map[0],
    // map[1], INTER_LINEAR) and crop.  xy / a: each view's CV_16SC2 / CV_16UC1 maps from initUndistortRectifyMap, cropped
    // to the context's W x H (map(cropBox)); src_width x src_height: the camera frames' size.  setInputImages then takes
    // CV_8UC3 frames of that size.  src_width = src_height = 0 with empty maps turns it off.
    int setRectify(const cv::Mat& lxy, const cv::Mat& la, const cv::Mat& rxy, const cv::Mat& ra, int src_width,
                   int src_height);
    int printCV(void);
    // OpenCV's reprojectImageTo3D(disp, xyz, Q, handleMissingValues) of one view's map (PSM_LEFT / PSM_RIGHT) on the
    // device, bit for bit (psm_read_points): xyz becomes H x W CV_32FC3 (X, Y, Z).  Q: the rig's 4 x 4 reprojection
    // matrix, row-major (stereoRectify's Q, the reference's camProps.Q).  postProcessed: the maps of the last
    // PostProcess_GPU, else those of the last DispSelect_GPU.
    int reprojectImageTo3D(cv::Mat& xyz, const double Q[16], bool handleMissingValues = false, int view = PSM_LEFT,
                           bool postProcessed = true);

    // GPU stages (the path behind the `m` toggle): 0 = success, as in the reference
    int CostConst_GPU();
    int CostFilter_GPU();
    int DispSelect_GPU();
    int PostProcess_GPU();

    // CPU stages are the reference's own code and are not part of this library
    int CostConst() { return not_built("CostConst"); }
    int CostConst_CPU() { return not_built("CostConst_CPU"); }
    int CostFilter() { return not_built("CostFilter"); }
    int CostFilter_CPU() { return not_built("CostFilter_CPU"); }
    int CostFilter_FGF() { return not_built("CostFilter_FGF"); }
    int DispSelect_CPU() { return not_built("DispSelect_CPU"); }
    int PostProcess_CPU() { return not_built("PostProcess_CPU"); }

    // stage timers of the last frame in ms (role of cvc_time/cvf_time/dispsel_time, StereoMatch.cpp:209-241)
    float stage_ms(int stage) const { float ms = -1.f; psm_stage_ms(ctx, stage, &ms); return ms; }
    const char* last_error() const { return psm_last_error(ctx); }

private:
    int not_built(const char* what) const
    {
        std::fprintf(stderr, "DispEst::%s: CPU stage not built into the GPU facade (use the reference's own)\n", what);
        return -1;
    }
    cv::Mat lImg, rImg;
    int hei, wid, maxDis, threads;
    bool useOCL;
    unsigned int subsample_rate = 4;
    int views = PSM_VIEWS_BOTH;
    int src_w = 0, src_h = 0;   // setRectify: the size of the frames CostConst_GPU takes, 0 = the context's
    int yuv_format = 0;         // setInputImagesYUV: the PSM_YUV_* format of lImg / rImg, 0 = BGR frames
    int bayer_pattern = 0;      // setInputImagesBayer: the PSM_BAYER_* pattern of lImg / rImg, 0 = not Bayer frames
    int bayer_method = PSM_DEMOSAIC_BILINEAR;
    bool cost_output = false;
    bool runner_up_output = false;
    int set_output(int key, bool on, bool& flag);
    int read_planes(int view, int n, int (*read)(psm_ctx*, int, float*, size_t), cv::Mat* planes);
    psm_ctx* ctx = nullptr;
};
