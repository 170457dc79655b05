// TEST INFRASTRUCTURE ONLY -- never part of the product path.
//
// C entry points that run the reference's OWN debug-image code on a given state and return the images it writes: the real
// Evaluator::evaluate with saving on (Evaluator.h:113-187: D, N, E) and PMStereoBase::viewConsistencyCheck (PMStereoBase.h:87-108: the two
// C images).  It is oracle/ref_run_driver.cpp (the reference's whole run over the mini cv:: layer of oracle/cvshim/) compiled once more with
// cv::imwrite redirected to a capturing function: the shim's own imwrite writes nothing, and every other driver keeps it.  Captured
// images are the Mats imwrite receives -- float for D and N (imwrite's 8-bit conversion is restated by oracle/vis_oracle.sat8 and pinned
// to cv2 separately), 8-bit for E and C.  Built by oracle/build_ref_vis.py into oracle/_ref/liblexp_ref_vis.so.
#include <opencv2/opencv.hpp>
#include <string>
#include <vector>

namespace cv {
inline std::vector<Mat>& lexp_vis_captured() { static std::vector<Mat> v; return v; }
inline bool lexp_vis_imwrite(const std::string&, const Mat& m) { lexp_vis_captured().push_back(m.clone()); return true; }
}  // namespace cv

#define imwrite lexp_vis_imwrite
#include "ref_run_driver.cpp"
#undef imwrite

namespace {

struct VisProbe : FastGCStereo {
    using FastGCStereo::FastGCStereo;
    using PMStereoBase::currentLabeling_;
    using PMStereoBase::currentLabeling_m_;
    using PMStereoBase::currentCost_;
    using PMStereoBase::stereoEnergy;
    using PMStereoBase::viewConsistencyCheck;
};

// the k-th captured image, copied row by row into out (elem bytes per pixel).  Images are told apart by their order, not their file
// names: Evaluator::evaluate passes its std::string header to cv::format's "%s", which g++ does not turn into a C string.
void copy_capture(size_t k, int H, int W, size_t elem, int type, void* out) {
    const std::vector<cv::Mat>& v = cv::lexp_vis_captured();
    if (k >= v.size()) throw std::runtime_error("fewer images written than expected");
    const cv::Mat& m = v[k];
    if (m.rows != H || m.cols != W || m.type() != type) throw std::runtime_error("captured image " + std::to_string(k) + ": unexpected size or type");
    for (int y = 0; y < H; y++) memcpy((char*)out + (size_t)y * W * elem, m.ptr<uchar>(y), (size_t)W * elem);
}

}  // namespace

extern "C" {

const char* ref_vis_last_error() { return g_err.c_str(); }

// Evaluator(dispGT, nonocc, 255 / max_disp, "result", log_dir)::evaluate(labeling_m, cost, energy, show off, save on, print off, index 7,
// mode) with setPrecision(precision) / setErrorThreshold(threshold), on the given labeling [H][W][4] of view `mode`.  Outputs the images it
// writes: d [H][W] and n [H][W][3] as the float Mats imwrite receives (disparityMapVis * 255, normalMapVis * 255), e [H][W] 8-bit.
int ref_vis_evaluate(int H, int W, const uchar* imL, const uchar* imR, float max_disp, const float* labeling, const float* gt, const uchar* nonocc,
                     float precision, float threshold, int mode, const char* log_dir, float* d, float* n, uchar* e) {
    try {
        VisProbe s(bgr(imL, H, W), bgr(imR, H, W), params(20, 1.0f), max_disp, 0, 0);
        cv::Mat(H, W, CV_32FC4, (void*)labeling).copyTo(s.currentLabeling_[mode]);
        Evaluator ev(f32(gt, H, W), u8(nonocc, H, W), 255.0f / max_disp, "result", log_dir, false, false, true);
        ev.setPrecision(precision);
        ev.setErrorThreshold(threshold);
        cv::lexp_vis_captured().clear();
        ev.evaluate(s.currentLabeling_m_[mode], s.currentCost_[mode], *s.stereoEnergy, false, true, false, 7, mode);
        if (cv::lexp_vis_captured().size() != 3) throw std::runtime_error("Evaluator::evaluate did not write three images");
        copy_capture(0, H, W, 4, CV_32FC1, d);    // Evaluator.h:164-166: D, N, E in this order
        copy_capture(1, H, W, 12, CV_32FC3, n);
        copy_capture(2, H, W, 1, CV_8UC1, e);
        return 0;
    } catch (const std::exception& ex) { g_err = ex.what(); return -1; }
}

// viewConsistencyCheck(check0, check1) of an optimiser with MIN min_disp / MAX max_disp whose currentLabeling_[0 / 1] are lab0 / lab1
// [H][W][4]: c0, c1 [H][W][3] 8-bit BGR.
int ref_vis_check(int H, int W, const uchar* imL, const uchar* imR, float min_disp, float max_disp, const float* lab0, const float* lab1, uchar* c0,
                  uchar* c1) {
    try {
        VisProbe s(bgr(imL, H, W), bgr(imR, H, W), params(20, 1.0f), max_disp, min_disp, 0);
        cv::Mat(H, W, CV_32FC4, (void*)lab0).copyTo(s.currentLabeling_[0]);
        cv::Mat(H, W, CV_32FC4, (void*)lab1).copyTo(s.currentLabeling_[1]);
        cv::Mat a, b;
        s.viewConsistencyCheck(a, b);
        cv::lexp_vis_captured().clear();
        cv::lexp_vis_imwrite("c0", a);   // as FastGCStereo.h:164-165 writes them
        cv::lexp_vis_imwrite("c1", b);
        copy_capture(0, H, W, 3, CV_8UC3, c0);
        copy_capture(1, H, W, 3, CV_8UC3, c1);
        return 0;
    } catch (const std::exception& ex) { g_err = ex.what(); return -1; }
}

}  // extern "C"
