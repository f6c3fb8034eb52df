// DispEstB200.cpp -- see DispEstB200.h.  Every method cites the reference code it stands in for.
#include "DispEstB200.h"

#include <cassert>
#include <cstring>

// reference src/DispEst.cpp:10-143: type check (exit(1) on mismatch), output maps, and -- instead of
// the OpenCL context / queue / 12 cl_mem buffers / three run-time compiled programs -- one psm_ctx.
DispEst::DispEst(cv::Mat l, cv::Mat r, const int d, int t, bool ocl, int block_slices, std::vector<int> devices, int min_disp)
    : lImg(l), rImg(r), maxDis(d), threads(t), useOCL(ocl)
{
    hei = lImg.rows;
    wid = lImg.cols;
    if (lImg.type() != rImg.type()) {
        std::printf("DE: Error - Left & Right images are of different types.\n");
        std::exit(1);
    }
    // maxDis > 256: 16-bit maps (psm_create_u16, maxDis <= 4096)
    const bool wide = maxDis > 256;
    lDisMap = cv::Mat::zeros(hei, wid, wide ? CV_16UC1 : CV_8UC1);
    rDisMap = cv::Mat::zeros(hei, wid, wide ? CV_16UC1 : CV_8UC1);
    lValid = cv::Mat::zeros(hei, wid, CV_8UC1);   // DispEst.cpp:48-49
    rValid = cv::Mat::zeros(hei, wid, CV_8UC1);
    if (useOCL) {
        const int dev = devices.empty() ? 0 : devices[0];
        if (devices.empty()) devices.push_back(dev);
        const int rc = min_disp > 0
                           ? psm_create_range(&ctx, wid, hei, min_disp, maxDis, devices.data(), (int)devices.size(),
                                              block_slices > 0 ? block_slices : 0, wide ? 16 : 8)
                     : devices.size() >= 2
                           ? psm_create_multi(&ctx, wid, hei, maxDis, devices.data(), (int)devices.size(), block_slices > 0 ? block_slices : 0,
                                              wide ? 16 : 8)
                     : block_slices > 0 ? psm_create_blocked(&ctx, wid, hei, maxDis, 0, maxDis, block_slices, wide ? 16 : 8, dev)
                     : wide ? psm_create_u16(&ctx, wid, hei, maxDis, 0, maxDis, dev) : psm_create(&ctx, wid, hei, maxDis, dev);
        if (rc != PSM_OK) {
            // reference logs OpenCL set-up failures and carries on (DispEst.cpp:69-79); so do we, with
            // the GPU stages then returning an error code instead of computing anything on the CPU
            std::fprintf(stderr, "Failed to create the GPU context: %s\n", psm_last_error(nullptr));
            ctx = nullptr;
        }
    }
}

// reference src/DispEst.cpp:145-162
DispEst::~DispEst(void)
{
    if (ctx) psm_destroy(ctx);
}

// reference src/DispEst.cpp:164-170
int DispEst::setInputImages(cv::Mat leftImg, cv::Mat rightImg)
{
    assert(leftImg.type() == rightImg.type());
    lImg = leftImg;
    rImg = rightImg;
    yuv_format = 0;
    bayer_pattern = 0;
    return 0;
}

int DispEst::setInputImagesYUV(cv::Mat leftImg, cv::Mat rightImg, int format)
{
    if (format < PSM_YUV_NV12 || format > PSM_YUV_YVYU) {
        std::fprintf(stderr, "DispEst::setInputImagesYUV: unknown format %d\n", format);
        return -1;
    }
    lImg = leftImg;
    rImg = rightImg;
    yuv_format = format;
    bayer_pattern = 0;
    return 0;
}

int DispEst::setInputImagesBayer(cv::Mat leftImg, cv::Mat rightImg, int pattern, int method)
{
    if (pattern < PSM_BAYER_RGGB || pattern > PSM_BAYER_GBRG || (method != PSM_DEMOSAIC_BILINEAR && method != PSM_DEMOSAIC_EA)) {
        std::fprintf(stderr, "DispEst::setInputImagesBayer: unknown pattern %d or method %d\n", pattern, method);
        return -1;
    }
    lImg = leftImg;
    rImg = rightImg;
    yuv_format = 0;
    bayer_pattern = pattern;
    bayer_method = method;
    return 0;
}

// reference src/DispEst.cpp:172-179
int DispEst::setThreads(unsigned int newThreads)
{
    if (newThreads > MAX_CPU_THREADS) return -1;
    threads = newThreads;
    return 0;
}

int DispEst::setGuidedFilter(int window, float eps)
{
    if (!ctx) return -1;
    return psm_set_guided_filter(ctx, window, eps);
}

int DispEst::setMatchingCost(float alpha, float tau_color, float tau_grad)
{
    if (!ctx) return -1;
    return psm_set_matching_cost(ctx, alpha, tau_color, tau_grad);
}

int DispEst::setPostFilter(int radius, float sigma, int iterations, int weight_type)
{
    if (!ctx) return -1;
    return psm_set_post_filter(ctx, radius, sigma, iterations, weight_type);
}

int DispEst::setLRCheck(int mode)
{
    if (!ctx) return -1;
    return psm_set_lr_check(ctx, mode);
}

int DispEst::setSpeckleFilter(int mode, int max_size, int max_diff)
{
    if (!ctx) return -1;
    return psm_set_speckle_filter(ctx, mode, max_size, max_diff);
}

int DispEst::setDisparityCheck(int mode, int max_diff)
{
    if (!ctx) return -1;
    return psm_set_disparity_check(ctx, mode, max_diff);
}

int DispEst::setUniquenessCheck(int mode, int ratio)
{
    if (!ctx) return -1;
    return psm_set_uniqueness_check(ctx, mode, ratio);
}

int DispEst::setMedianBlur(int mode, int ksize)
{
    if (!ctx) return -1;
    return psm_set_median_blur(ctx, mode, ksize);
}

int DispEst::setViews(int v)
{
    if (!ctx) return -1;
    const int rc = psm_set_option(ctx, PSM_OPT_VIEWS, v);
    if (rc == PSM_OK) views = v;
    return rc;
}

int DispEst::setCostOutput(bool on) { return set_output(PSM_OPT_COSTS, on, cost_output); }

int DispEst::setRunnerUpOutput(bool on) { return set_output(PSM_OPT_RUNNER_UP, on, runner_up_output); }

// a per-pixel output's option `key` = on; `flag` (what DispSelect_GPU reads) follows it where the context accepts it
int DispEst::set_output(int key, bool on, bool& flag)
{
    if (!ctx) return -1;
    const int rc = psm_set_option(ctx, key, on ? 1 : 0);
    if (rc == PSM_OK) flag = on;
    return rc;
}

// one view's n planes (read: psm_read_costs or psm_read_runner_up, contiguous) -> n CV_32FC1 matrices
int DispEst::read_planes(int view, int n, int (*read)(psm_ctx*, int, float*, size_t), cv::Mat* planes)
{
    cv::Mat all(n * hei, wid, CV_32FC1);
    if (int rc = read(ctx, view, all.ptr<float>(), all.step)) return rc;
    for (int k = 0; k < n; ++k) {
        planes[k] = cv::Mat(hei, wid, CV_32FC1);
        for (int y = 0; y < hei; ++y) std::memcpy(planes[k].ptr<float>(y), all.ptr<float>(k * hei + y), (size_t)wid * sizeof(float));
    }
    return 0;
}

// reference src/StereoMatch.cpp:149-153 (remap of each camera frame, then the crop) as a device step of CostConst_GPU
int DispEst::setRectify(const cv::Mat& lxy, const cv::Mat& la, const cv::Mat& rxy, const cv::Mat& ra, int src_width,
                        int src_height)
{
    if (!ctx) return -1;
    if (!src_width && !src_height && lxy.empty() && la.empty() && rxy.empty() && ra.empty()) {
        const int rc = psm_set_rectify(ctx, 0, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0);
        if (rc == PSM_OK) src_w = src_h = 0;
        return rc;
    }
    for (const cv::Mat* m : {&lxy, &la, &rxy, &ra})
        if (m->rows != hei || m->cols != wid || m->type() != (m == &lxy || m == &rxy ? CV_16SC2 : CV_16UC1)) {
            std::fprintf(stderr, "DispEst::setRectify: the maps must be %dx%d CV_16SC2 (xy) and CV_16UC1 (a), cropped to "
                                 "the disparity maps' size\n", wid, hei);
            return -1;
        }
    const int rc = psm_set_rectify(ctx, src_width, src_height, lxy.ptr<int16_t>(), lxy.step, la.ptr<uint16_t>(), la.step,
                                   rxy.ptr<int16_t>(), rxy.step, ra.ptr<uint16_t>(), ra.step);
    if (rc == PSM_OK) { src_w = src_width; src_h = src_height; }
    return rc;
}

// reference src/DispEst.cpp:181-194 dumps every slice as PNG; here: slice statistics on stdout
int DispEst::reprojectImageTo3D(cv::Mat& xyz, const double Q[16], bool handleMissingValues, int view, bool postProcessed)
{
    if (!ctx) return -1;
    if (xyz.rows != hei || xyz.cols != wid || xyz.type() != CV_32FC3 || !xyz.data) xyz.create(hei, wid, CV_32FC3);
    return psm_read_points(ctx, postProcessed ? 1 : 0, view, Q, handleMissingValues ? 1 : 0, xyz.ptr<float>(), xyz.step);
}

int DispEst::printCV(void)
{
    if (!ctx) return -1;
    cv::Mat s(hei, wid, CV_32FC1);
    for (int v = 0; v < 2; ++v)
        for (int i = 0; i < maxDis; ++i) {
            if (int rc = psm_read_cost_slice(ctx, v, i, s.ptr<float>(), s.step)) return rc;
            double sum = 0;
            for (int y = 0; y < hei; ++y)
                for (int x = 0; x < wid; ++x) sum += s.ptr<float>(y)[x];
            std::printf("%cCV%d mean %.6f\n", v ? 'r' : 'l', i, sum / ((double)hei * wid));
        }
    return 0;
}

// reference src/DispEst.cpp:272-276 -> CVC_cl::buildCV (src/CVC_cl.cpp:93-211): upload + build both volumes
int DispEst::CostConst_GPU()
{
    if (!ctx) return -1;
    // the context was sized at construction: a differently shaped or typed Mat from setInputImages must not reach
    // the 2-D copy (the reference re-creates DispEst on every dataset change, StereoMatch.cpp:601-602)
    // with setRectify on, the frames are the camera's (src_w x src_h, 8-bit)
    const int fw = src_w ? src_w : wid, fh = src_w ? src_h : hei;
    if (yuv_format) {
        const bool is420 = yuv_format <= PSM_YUV_YV12;
        const int rows = is420 ? fh / 2 * 3 : fh, type = is420 ? CV_8UC1 : CV_8UC2;
        for (const cv::Mat* m : {&lImg, &rImg})
            if (m->rows != rows || m->cols != fw || m->type() != type) {
                std::fprintf(stderr, "DispEst::CostConst_GPU: YUV frames must be %dx%d %s\n", fw, rows,
                             is420 ? "CV_8UC1" : "CV_8UC2");
                return -1;
            }
        if (int rc = psm_set_images_yuv(ctx, yuv_format, lImg.ptr<uint8_t>(), lImg.step, rImg.ptr<uint8_t>(), rImg.step))
            return rc;
        return psm_cost_const(ctx);
    }
    if (bayer_pattern) {
        for (const cv::Mat* m : {&lImg, &rImg})
            if (m->rows != fh || m->cols != fw || m->type() != CV_8UC1) {
                std::fprintf(stderr, "DispEst::CostConst_GPU: Bayer frames must be %dx%d CV_8UC1\n", fw, fh);
                return -1;
            }
        if (int rc = psm_set_images_bayer(ctx, bayer_pattern, bayer_method, lImg.ptr<uint8_t>(), lImg.step,
                                          rImg.ptr<uint8_t>(), rImg.step))
            return rc;
        return psm_cost_const(ctx);
    }
    if (lImg.rows != fh || lImg.cols != fw || rImg.rows != fh || rImg.cols != fw || lImg.type() != rImg.type() ||
        lImg.channels() != 3) {
        std::fprintf(stderr, "DispEst::CostConst_GPU: input images must be %dx%d, 3 channels, equal types\n", fw, fh);
        return -1;
    }
    int rc;
    if ((lImg.type() & CV_MAT_DEPTH_MASK) == CV_32F)
        rc = psm_set_images(ctx, lImg.ptr<float>(), lImg.step, rImg.ptr<float>(), rImg.step);
    else
        rc = psm_set_images_u8(ctx, lImg.ptr<uint8_t>(), lImg.step, rImg.ptr<uint8_t>(), rImg.step);
    if (rc) return rc;
    return psm_cost_const(ctx);
}

// reference src/DispEst.cpp:299-308 -> CVF_cl::preprocess + CVF_cl::filterCV per view
int DispEst::CostFilter_GPU()
{
    if (!ctx) return -1;
    return psm_cost_filter(ctx);
}

// reference src/DispEst.cpp:323-328 -> DispSel_cl::CVSelect (src/DispSel_cl.cpp:69-139)
int DispEst::DispSelect_GPU()
{
    if (!ctx) return -1;
    const bool both = views == PSM_VIEWS_BOTH;   // a left-only context takes no right map
    const int rc = lDisMap.type() == CV_16UC1
        ? psm_disp_select_u16(ctx, lDisMap.ptr<uint16_t>(), lDisMap.step, both ? rDisMap.ptr<uint16_t>() : nullptr, rDisMap.step)
        : psm_disp_select(ctx, lDisMap.ptr<uint8_t>(), lDisMap.step, both ? rDisMap.ptr<uint8_t>() : nullptr, rDisMap.step);
    if (rc) return rc;
    if (cost_output) {
        if (int e = read_planes(PSM_LEFT, 3, psm_read_costs, lCosts)) return e;
        if (both)
            if (int e = read_planes(PSM_RIGHT, 3, psm_read_costs, rCosts)) return e;
    }
    if (runner_up_output) {
        if (int e = read_planes(PSM_LEFT, 2, psm_read_runner_up, lRunnerUp)) return e;
        if (both)
            if (int e = read_planes(PSM_RIGHT, 2, psm_read_runner_up, rRunnerUp)) return e;
    }
    return 0;
}

// reference src/DispEst.cpp:338-344 -> PP::processDM (src/PP.cpp:402-425): the joint weighted-median filter of
// both maps, after the left-right check and fill that setLRCheck enables (PP.cpp:405-406, psm_lr.cuh) and the speckle
// removal, disparity check, uniqueness test and median that setSpeckleFilter, setDisparityCheck, setUniquenessCheck and
// setMedianBlur enable (psm_speckle.cuh, psm_dcheck.cuh, psm_unique.cuh, psm_median.cuh).  The reference runs it on the
// CPU even in GPU mode; here it is a device stage (psm_pp.cuh).  The masks exist only where the check ran (the context
// answers PSM_ESTATE otherwise), the right one only on a two-view context.
int DispEst::PostProcess_GPU()
{
    if (!ctx) return -1;
    const bool both = views == PSM_VIEWS_BOTH;
    const int rc = lDisMap.type() == CV_16UC1
        ? psm_post_process_u16(ctx, lDisMap.ptr<uint16_t>(), lDisMap.step, both ? rDisMap.ptr<uint16_t>() : nullptr, rDisMap.step)
        : psm_post_process(ctx, lDisMap.ptr<uint8_t>(), lDisMap.step, both ? rDisMap.ptr<uint8_t>() : nullptr, rDisMap.step);
    if (rc) return rc;
    const int e = psm_read_valid_mask(ctx, PSM_LEFT, lValid.ptr<uint8_t>(), lValid.step);
    if (e == PSM_ESTATE) return 0;   // the check did not run
    if (e) return e;
    return both ? psm_read_valid_mask(ctx, PSM_RIGHT, rValid.ptr<uint8_t>(), rValid.step) : 0;
}
