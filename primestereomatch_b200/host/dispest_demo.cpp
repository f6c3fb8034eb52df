// dispest_demo.cpp -- drives the C++ DispEst facade exactly like StereoMatch::compute does
// (reference src/StereoMatch.cpp:198-241): setInputImages -> CostConst_GPU -> CostFilter_GPU ->
// DispSelect_GPU -> PostProcess_GPU.  Raw I/O so it needs no image library:
//   dispest_demo W H D left.f32 right.f32 out_left.u8 out_right.u8 [window eps [alpha tau_color tau_grad
//                [radius sigma iterations weight [lr_mode]]]]
// The optional window / eps go to setGuidedFilter (default: the reference's 8 and 0.0001f), the optional alpha and
// thresholds to setMatchingCost (default: 0.9 inf inf, i.e. no truncation), the optional post-filter radius, sigma,
// iterations and weight (exp, iv1, iv2 or off) to setPostFilter (default: 9 25.5 1 exp), the optional left-right check
// mode (0 off, 1 check + fill + post-filter, 2 check + fill) to setLRCheck (default 0).  D up to 4096: above 256 the
// maps are CV_16UC1 and the output files hold 2-byte (native-endian uint16) disparities.  A leading
// `--block-slices N` runs a blocked context (psm_create_blocked) that holds N disparity slices at a time, a leading
// `--devices 0,1,...` a context over those CUDA devices (two or more ids: psm_create_multi; ids may repeat), a leading
// `--min-disp N` a context over disparities [N, D) alone (psm_create_range; the maps hold absolute disparities), a
// leading `--speckle MODE SIZE DIFF` speckle removal (setSpeckleFilter: MODE 0 off, 1 first, 2 only), a leading
// `--disp-check MODE MAXDIFF` the one-view disparity check (setDisparityCheck: MODE 0 off, 1 first, 2 only; it turns
// setCostOutput on, which the check reads), a leading `--uniqueness MODE RATIO` the uniqueness test
// (setUniquenessCheck: MODE 0 off, 1 first, 2 only; it turns setCostOutput and setRunnerUpOutput on, which the test
// reads), a leading `--median MODE KSIZE` the median (setMedianBlur: MODE 0 off, 1 first, 2 only; KSIZE 3 or 5), a leading
// `--points Q.f64 out.xyz` the left view's 3D points of the final maps (reprojectImageTo3D with the 16 native-endian
// doubles of Q.f64, row-major): out.xyz holds H x W x 3 native float32 X, Y, Z.  A leading
// `--left-only` computes the left map alone (setViews(PSM_VIEWS_LEFT)) and writes no right map: outR is not created.  A
// leading `--rectify SW SH left.map right.map` rectifies raw camera frames on the device (setRectify): each .map file
// holds W x H native-endian int16 pairs (map[0], CV_16SC2), then W x H uint16 (map[1], CV_16UC1), both cropped to W x H,
// and left / right are then 8-bit BGR frames of SW x SH instead of float frames of W x H.  A leading `--yuv FORMAT`
// (nv12, nv21, i420, yv12, yuyv, uyvy or yvyu) reads left / right as raw YUV frames in cv2's layout of W x H (or SW x SH
// with --rectify): (H * 3 / 2) rows of W bytes for the 4:2:0 formats, H rows of 2 * W bytes for the 4:2:2 ones, converted
// to BGR on the device (setInputImagesYUV).  A leading `--bayer PATTERN` (rggb, bggr, grbg or gbrg) reads left / right
// as Bayer raw frames of W x H (or SW x SH with --rectify), H rows of W bytes, demosaiced on the device
// (setInputImagesBayer) as cvtColor(COLOR_Bayer<PATTERN>2BGR) does, or as _EA with a following `--ea`.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "DispEstB200.h"

static bool read_all(const char* path, void* dst, size_t n)
{
    FILE* f = std::fopen(path, "rb");
    if (!f) return false;
    const size_t got = std::fread(dst, 1, n, f);
    std::fclose(f);
    return got == n;
}

int main(int argc, char** argv)
{
    int block_slices = 0, min_disp = 0;
    int speckle[3] = {0, 0, 0};   // mode, max_size, max_diff
    int dcheck[2] = {0, 1};       // mode, max_diff
    int unique[2] = {0, 10};      // mode, ratio
    int median[2] = {0, 3};       // mode, ksize
    const char* points[2] = {nullptr, nullptr};   // Q file, output file
    int src_size[2] = {0, 0};                     // --rectify: SW, SH
    const char* map_files[2] = {nullptr, nullptr};
    int yuv = 0;                                  // --yuv: PSM_YUV_* of the frames, 0 = BGR
    int bayer = 0, demosaic = PSM_DEMOSAIC_BILINEAR;   // --bayer: PSM_BAYER_* of the frames, 0 = not Bayer; --ea
    std::vector<int> devices;
    const bool left_only = argc >= 2 && !std::strcmp(argv[1], "--left-only");
    if (left_only) {
        argv[1] = argv[0];
        ++argv;
        --argc;
    }
    while (argc >= 3 && (!std::strcmp(argv[1], "--block-slices") || !std::strcmp(argv[1], "--devices") ||
                         !std::strcmp(argv[1], "--min-disp") || !std::strcmp(argv[1], "--speckle") ||
                         !std::strcmp(argv[1], "--disp-check") || !std::strcmp(argv[1], "--uniqueness") ||
                         !std::strcmp(argv[1], "--median") ||
                         !std::strcmp(argv[1], "--points") || !std::strcmp(argv[1], "--rectify") ||
                         !std::strcmp(argv[1], "--yuv") || !std::strcmp(argv[1], "--bayer") ||
                         !std::strcmp(argv[1], "--ea"))) {
        if (!std::strcmp(argv[1], "--ea")) {
            demosaic = PSM_DEMOSAIC_EA;
            argv[1] = argv[0];
            ++argv;
            --argc;
            continue;
        }
        if (!std::strcmp(argv[1], "--bayer")) {
            static const char* const names[] = {"rggb", "bggr", "grbg", "gbrg"};
            for (int k = 0; k < 4; ++k)
                if (!std::strcmp(argv[2], names[k])) bayer = PSM_BAYER_RGGB + k;
            if (!bayer) { std::fprintf(stderr, "unknown --bayer pattern %s\n", argv[2]); return 2; }
            argv[2] = argv[0];
            argv += 2;
            argc -= 2;
            continue;
        }
        if (!std::strcmp(argv[1], "--yuv")) {
            static const char* const names[] = {"nv12", "nv21", "i420", "yv12", "yuyv", "uyvy", "yvyu"};
            for (int k = 0; k < 7; ++k)
                if (!std::strcmp(argv[2], names[k])) yuv = PSM_YUV_NV12 + k;
            if (!yuv) { std::fprintf(stderr, "unknown --yuv format %s\n", argv[2]); return 2; }
            argv[2] = argv[0];
            argv += 2;
            argc -= 2;
            continue;
        }
        if (!std::strcmp(argv[1], "--rectify")) {
            if (argc < 6) break;
            src_size[0] = std::atoi(argv[2]);
            src_size[1] = std::atoi(argv[3]);
            map_files[0] = argv[4];
            map_files[1] = argv[5];
            argv[5] = argv[0];
            argv += 5;
            argc -= 5;
            continue;
        }
        if (!std::strcmp(argv[1], "--points")) {
            if (argc < 4) break;
            points[0] = argv[2];
            points[1] = argv[3];
            argv[3] = argv[0];
            argv += 3;
            argc -= 3;
            continue;
        }
        if (!std::strcmp(argv[1], "--disp-check") || !std::strcmp(argv[1], "--uniqueness") ||
            !std::strcmp(argv[1], "--median")) {
            if (argc < 4) break;
            int* const dst = argv[1][2] == 'd' ? dcheck : argv[1][2] == 'u' ? unique : median;
            dst[0] = std::atoi(argv[2]);
            dst[1] = std::atoi(argv[3]);
            argv[3] = argv[0];
            argv += 3;
            argc -= 3;
            continue;
        }
        if (!std::strcmp(argv[1], "--speckle")) {
            if (argc < 5) break;
            for (int k = 0; k < 3; ++k) speckle[k] = std::atoi(argv[2 + k]);
            argv[4] = argv[0];
            argv += 4;
            argc -= 4;
            continue;
        }
        if (!std::strcmp(argv[1], "--block-slices")) {
            block_slices = std::atoi(argv[2]);
        } else if (!std::strcmp(argv[1], "--min-disp")) {
            min_disp = std::atoi(argv[2]);
        } else {
            for (const char* p = argv[2]; *p;) {
                char* end = nullptr;
                devices.push_back((int)std::strtol(p, &end, 10));
                if (end == p) { std::fprintf(stderr, "bad device list %s\n", argv[2]); return 2; }
                p = *end == ',' ? end + 1 : end;
            }
        }
        argv[2] = argv[0];
        argv += 2;
        argc -= 2;
    }
    if (argc != 8 && argc != 10 && argc != 13 && argc != 17 && argc != 18) {
        std::fprintf(stderr, "usage: %s [--left-only] [--block-slices N] [--devices i,j,...] [--min-disp N] [--speckle MODE SIZE DIFF] [--disp-check MODE MAXDIFF] [--uniqueness MODE RATIO] [--median MODE KSIZE] [--points Q.f64 out.xyz] [--rectify SW SH left.map right.map] [--yuv FORMAT | --bayer PATTERN [--ea]] W H D left.f32 right.f32 outL.u8 outR.u8 [window eps [alpha tau_color tau_grad"
                             " [radius sigma iterations exp|iv1|iv2|off [lr_mode]]]]\n", argv[0]);
        return 2;
    }
    const int W = std::atoi(argv[1]), H = std::atoi(argv[2]), D = std::atoi(argv[3]);
    if (b200devicepoll() == 0) { std::fprintf(stderr, "no CUDA device\n"); return 3; }
    // the frames: float W x H, or with --rectify the camera's 8-bit SW x SH
    const bool rectify = map_files[0] != nullptr;
    const int fw = rectify ? src_size[0] : W, fh = rectify ? src_size[1] : H;
    if (fw < 1 || fh < 1) { std::fprintf(stderr, "bad --rectify source size\n"); return 2; }
    if (yuv && bayer) { std::fprintf(stderr, "--yuv and --bayer: the frames are one or the other\n"); return 2; }
    // with --yuv: CV_8UC1 of (fh * 3 / 2) x fw (4:2:0) or CV_8UC2 of fh x fw (4:2:2); with --bayer: CV_8UC1 of fh x fw
    const int type = bayer ? CV_8UC1 : yuv ? (yuv <= PSM_YUV_YV12 ? CV_8UC1 : CV_8UC2) : rectify ? CV_8UC3 : CV_32FC3;
    const int rows = yuv && yuv <= PSM_YUV_YV12 ? fh / 2 * 3 : fh;
    cv::Mat l(rows, fw, type), r(rows, fw, type);
    if (!read_all(argv[4], l.data, l.step * rows) || !read_all(argv[5], r.data, r.step * rows)) { std::fprintf(stderr, "bad input\n"); return 2; }
    const bool framed = rectify || yuv || bayer;   // the frames do not give the context's size
    cv::Mat sized(H, W, framed ? CV_8UC3 : l.type());   // the facade takes the context's size from its first frames
    DispEst* SMDE = new DispEst(framed ? sized : l, framed ? sized : r, D, MAX_CPU_THREADS, true, block_slices, devices,
                                min_disp);
    if (bayer)
        SMDE->setInputImagesBayer(l, r, bayer, demosaic);
    else if (yuv)
        SMDE->setInputImagesYUV(l, r, yuv);
    else
        SMDE->setInputImages(l, r);
    SMDE->setThreads(MAX_CPU_THREADS);
    SMDE->setSubsampleRate(4);
    int rc = left_only ? SMDE->setViews(PSM_VIEWS_LEFT) : 0;
    if (!rc && rectify) {
        cv::Mat xy[2], a[2];
        for (int v = 0; v < 2; ++v) {
            xy[v].create(H, W, CV_16SC2);
            a[v].create(H, W, CV_16UC1);
            FILE* f = std::fopen(map_files[v], "rb");
            const bool ok = f && std::fread(xy[v].data, 1, xy[v].step * H, f) == xy[v].step * H &&
                            std::fread(a[v].data, 1, a[v].step * H, f) == a[v].step * H;
            if (f) std::fclose(f);
            if (!ok) { std::fprintf(stderr, "bad map file %s\n", map_files[v]); return 2; }
        }
        rc = SMDE->setRectify(xy[0], a[0], xy[1], a[1], fw, fh);
    }
    if (!rc && argc >= 10) rc = SMDE->setGuidedFilter(std::atoi(argv[8]), (float)std::atof(argv[9]));
    if (!rc && argc >= 13)
        rc = SMDE->setMatchingCost((float)std::atof(argv[10]), (float)std::atof(argv[11]), (float)std::atof(argv[12]));
    if (!rc && argc >= 17) {
        const char* w = argv[16];
        const int wt = !std::strcmp(w, "exp") ? PSM_WMF_EXP : !std::strcmp(w, "iv1") ? PSM_WMF_IV1
                     : !std::strcmp(w, "iv2") ? PSM_WMF_IV2 : !std::strcmp(w, "off") ? PSM_WMF_OFF : -1;
        rc = SMDE->setPostFilter(std::atoi(argv[13]), (float)std::atof(argv[14]), std::atoi(argv[15]), wt);
    }
    if (!rc && argc == 18) rc = SMDE->setLRCheck(std::atoi(argv[17]));
    if (!rc && speckle[0]) rc = SMDE->setSpeckleFilter(speckle[0], speckle[1], speckle[2]);
    if (!rc && dcheck[0]) rc = SMDE->setDisparityCheck(dcheck[0], dcheck[1]);
    if (!rc && unique[0]) rc = SMDE->setUniquenessCheck(unique[0], unique[1]);
    if (!rc && median[0]) rc = SMDE->setMedianBlur(median[0], median[1]);
    if (!rc && (dcheck[0] || unique[0])) rc = SMDE->setCostOutput(true);
    if (!rc && unique[0]) rc = SMDE->setRunnerUpOutput(true);
    if (!rc) rc = SMDE->CostConst_GPU();
    if (!rc) rc = SMDE->CostFilter_GPU();
    if (!rc) rc = SMDE->DispSelect_GPU();
    if (!rc) rc = SMDE->PostProcess_GPU();
    cv::Mat xyz;
    if (!rc && points[0]) {
        double Q[16];
        if (!read_all(points[0], Q, sizeof Q)) { std::fprintf(stderr, "bad Q file %s\n", points[0]); return 2; }
        rc = SMDE->reprojectImageTo3D(xyz, Q);
    }
    if (rc) { std::fprintf(stderr, "stage failed (%d): %s\n", rc, SMDE->last_error()); return 1; }
    std::printf("CVC %.3f ms  CVF %.3f ms  DispSel %.3f ms  PP %.3f ms\n", SMDE->stage_ms(1), SMDE->stage_ms(2), SMDE->stage_ms(3), SMDE->stage_ms(5));
    const size_t bytes = SMDE->lDisMap.step * H;   // dense rows: W * 1 or W * 2 bytes
    FILE* f = std::fopen(argv[6], "wb"); std::fwrite(SMDE->lDisMap.data, 1, bytes, f); std::fclose(f);
    if (!left_only) { f = std::fopen(argv[7], "wb"); std::fwrite(SMDE->rDisMap.data, 1, bytes, f); std::fclose(f); }
    if (points[1]) { f = std::fopen(points[1], "wb"); std::fwrite(xyz.data, 1, xyz.step * H, f); std::fclose(f); }
    delete SMDE;
    return 0;
}
