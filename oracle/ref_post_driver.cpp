// TEST INFRASTRUCTURE ONLY -- never part of the product path.
//
// C entry points around the reference's OWN post-processing of a two-view run, PMStereoBase::postProcess and doConsistencyCheck
// (PMStereoBase.h:111-256), compiled from the reference's headers where they lie over the mini cv:: layer of oracle/cvshim/ (see
// oracle/build_ref_post.py).  Nothing here restates the algorithm.  The only cv:: call of that path the shim does not implement is
// cv::dilate; it is supplied below for what postProcess uses (CV_8UC1, the default 3x3 rectangle, the default border value) and
// substituted for the shim's stub inside the reference's headers only.  Output: oracle/_ref/liblexp_ref_post.so.
#include <opencv2/opencv.hpp>

namespace cv {
// cv::dilate(src, dst, cv::Mat()) on CV_8UC1: the maximum over the 3x3 neighbourhood; pixels outside the image never contribute
// (morphologyDefaultBorderValue is the identity of the maximum)
inline void lexp_dilate_3x3(const Mat& src, const OutputArray& dst, const Mat& kernel) {
    if (src.type() != CV_8UC1 || !kernel.empty()) shim_fail("dilate: only CV_8UC1 with the default kernel");
    Mat r(src.rows, src.cols, CV_8UC1);
    for (int y = 0; y < src.rows; y++)
        for (int x = 0; x < src.cols; x++) {
            uchar m = 0;
            for (int yy = std::max(y - 1, 0); yy <= std::min(y + 1, src.rows - 1); yy++)
                for (int xx = std::max(x - 1, 0); xx <= std::min(x + 1, src.cols - 1); xx++) m = std::max(m, src.at<uchar>(yy, xx));
            r.at<uchar>(y, x) = m;
        }
    dst.assign(r);
}
}  // namespace cv
#define dilate lexp_dilate_3x3
#include "Utilities.hpp"
#include "Plane.h"
#include "StereoEnergy.h"
#include "FastGCStereo.h"
#undef dilate
#include <omp.h>

namespace {

// the reference's optimiser with its protected post-processing and state opened up (nothing overridden)
struct PostProbe : FastGCStereo {
    using FastGCStereo::FastGCStereo;
    using PMStereoBase::postProcess;
    using PMStereoBase::doConsistencyCheck;
    using PMStereoBase::currentLabeling_;
};

thread_local std::string g_err;

void copy_in(const float* src, cv::Mat& dst, int H, int W) { cv::Mat(H, W, CV_32FC4, (void*)src).copyTo(dst); }
void copy_out(const cv::Mat& src, float* dst, int H, int W) {
    for (int y = 0; y < H; y++) memcpy(dst + (size_t)y * W * 4, src.ptr<float>(y), (size_t)W * 4 * sizeof(float));
}

}  // namespace

extern "C" {

const char* ref_post_last_error() { return g_err.c_str(); }
int ref_post_max_threads() { return omp_get_max_threads(); }

// The optimiser of a two-view run on 8-bit BGR images [H][W][3] with Parameters::windR / omega (its energy is the NaiveStereoEnergy
// PMStereoBase constructs, PMStereoBase.h:37: postProcess uses only its computeDisparities and computePatchWeight).
void* ref_post_create(int H, int W, const uchar* imL, const uchar* imR, int windR, float omega, float max_disp) {
    try {
        cv::Mat L = cv::Mat(H, W, CV_8UC3, (void*)imL).clone(), R = cv::Mat(H, W, CV_8UC3, (void*)imR).clone();
        Parameters params(20.f, windR, "GF", 1e-4f);
        params.omega = omega;
        return new PostProbe(L, R, params, max_disp, 0.f);
    } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
void ref_post_destroy(void* h) { delete (PostProbe*)h; }

// postProcess(currentLabeling_[0], currentLabeling_[1], threshold) (FastGCStereo.h:199-217 passes 1.5) on the labelings
// lab0 / lab1 [H][W][4], which receive the result.  nthreads > 0: OpenMP threads of its two parallel loops.
int ref_post_process(void* h, float* lab0, float* lab1, int H, int W, float threshold, int nthreads) {
    try {
        PostProbe& s = *(PostProbe*)h;
        copy_in(lab0, s.currentLabeling_[0], H, W);
        copy_in(lab1, s.currentLabeling_[1], H, W);
        if (nthreads > 0) omp_set_num_threads(nthreads);
        s.postProcess(s.currentLabeling_[0], s.currentLabeling_[1], threshold);
        copy_out(s.currentLabeling_[0], lab0, H, W);
        copy_out(s.currentLabeling_[1], lab1, H, W);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// doConsistencyCheck(disp0, disp1, fail0, fail1, threshold) on disparity maps [H][W]: fail uint8 [2][H][W]
int ref_consistency_check(void* h, const float* disp0, const float* disp1, int H, int W, float threshold, uchar* fail) {
    try {
        PostProbe& s = *(PostProbe*)h;
        cv::Mat f[2];
        s.doConsistencyCheck(cv::Mat(H, W, CV_32F, (void*)disp0), cv::Mat(H, W, CV_32F, (void*)disp1), f[0], f[1], threshold);
        for (int i = 0; i < 2; i++)
            for (int y = 0; y < H; y++) memcpy(fail + ((size_t)i * H + y) * W, f[i].ptr<uchar>(y), (size_t)W);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// cvutils::io::save_pfm_file (Utilities.hpp:84-137) of a float image [H][W]: the reference's disp0.pfm writer (main.cpp:319,410)
int ref_post_save_pfm(const char* path, const float* img, int H, int W) {
    try { cvutils::io::save_pfm_file(path, cv::Mat(H, W, CV_32F, (void*)img)); return 0; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

}  // extern "C"
