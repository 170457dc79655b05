// TEST INFRASTRUCTURE ONLY -- never part of the product path.
//
// C entry points around the reference's OWN whole run: FastGCStereo::run (FastGCStereo.h:133-222) with its random start
// (selectRandomPixelInRect + StereoEnergy::createRandomLabel) and the real Evaluator (Evaluator.h), compiled from the reference's headers
// where they lie over the mini cv:: layer of oracle/cvshim/ (see oracle/build_ref_run.py).  Nothing here restates the algorithm.  The
// Evaluator's window calls (namedWindow / imshow / waitKey) are stubbed below, RansacProposer's cv::solve is supplied; the shim's imwrite writes nothing.  The cv::dilate of
// postProcess is the one of oracle/ref_post_driver.cpp.  The Evaluator's mask expressions (`<=` and `!=` against a scalar, `&`, `|` of two 8-bit
// masks) are supplied below in the shim's own style: compare_ in double, bitwise operations per element.  Output: oracle/_ref/liblexp_ref_run.so.
#include <opencv2/opencv.hpp>
#include <iostream>

namespace cv {
inline Mat operator<=(const Mat& a, double s) { return compare_(a, s, [](double x, double y) { return x <= y; }); }
inline Mat operator!=(const Mat& a, double s) { return compare_(a, s, [](double x, double y) { return x != y; }); }
template <class Op> inline Mat bitwise8(const Mat& a, const Mat& b, Op op) {
    check_same(a, b);
    if (a.depth() != CV_8U) shim_fail("bitwise operation on non-8U");
    Mat r(a.rows, a.cols, a.type());
    const int n = a.cols * a.channels();
    for (int y = 0; y < a.rows; y++) { const uchar* p = a.ptr<uchar>(y); const uchar* q = b.ptr<uchar>(y); uchar* o = r.ptr<uchar>(y); for (int i = 0; i < n; i++) o[i] = op(p[i], q[i]); }
    return r;
}
inline Mat operator&(const Mat& a, const Mat& b) { return bitwise8(a, b, [](uchar x, uchar y) { return (uchar)(x & y); }); }
inline Mat operator|(const Mat& a, const Mat& b) { return bitwise8(a, b, [](uchar x, uchar y) { return (uchar)(x | y); }); }
enum { WINDOW_NORMAL = 0, WINDOW_KEEPRATIO = 0 };
inline void namedWindow(const std::string&, int = 0) {}
inline void imshow(const std::string&, const Mat&) {}
inline int waitKey(int = 0) { return -1; }
// cv::solve(A, b, x, DECOMP_SVD) of RansacProposer (3 unknowns; the shim's stub refuses it): the minimum-norm least-squares solution in
// double, from the cyclic Jacobi eigen-decomposition of A^T A (eigenvalues below 1e-12 of the largest count as zero).  The whole-run
// accuracy it serves does not depend on the last bits of a plane fit.
inline bool lexp_run_solve(const Mat& A, const Mat& b, const OutputArray& dst, int flags) {
    if (flags != DECOMP_SVD || A.type() != CV_32FC1 || b.type() != CV_32FC1 || A.cols != 3 || b.rows != A.rows) shim_fail("solve: only the RANSAC systems");
    double G[3][3] = {{0}}, g[3] = {0, 0, 0}, V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int r = 0; r < A.rows; r++)
        for (int i = 0; i < 3; i++) {
            g[i] += (double)A.at<float>(r, i) * (double)b.at<float>(r, 0);
            for (int j = 0; j < 3; j++) G[i][j] += (double)A.at<float>(r, i) * (double)A.at<float>(r, j);
        }
    for (int sweep = 0; sweep < 50; sweep++)
        for (int p = 0; p < 2; p++)
            for (int q = p + 1; q < 3; q++) {
                if (G[p][q] == 0.0) continue;
                const double th = 0.5 * std::atan2(2 * G[p][q], G[q][q] - G[p][p]), c = std::cos(th), s = std::sin(th);
                for (int k = 0; k < 3; k++) { const double a = G[k][p], d = G[k][q]; G[k][p] = c * a - s * d; G[k][q] = s * a + c * d; }
                for (int k = 0; k < 3; k++) { const double a = G[p][k], d = G[q][k]; G[p][k] = c * a - s * d; G[q][k] = s * a + c * d; }
                for (int k = 0; k < 3; k++) { const double a = V[k][p], d = V[k][q]; V[k][p] = c * a - s * d; V[k][q] = s * a + c * d; }
            }
    const double emax = std::max(std::fabs(G[0][0]), std::max(std::fabs(G[1][1]), std::fabs(G[2][2])));
    double x[3] = {0, 0, 0};
    for (int e = 0; e < 3; e++) {
        if (!(std::fabs(G[e][e]) > 1e-12 * emax)) continue;
        const double t = (V[0][e] * g[0] + V[1][e] * g[1] + V[2][e] * g[2]) / G[e][e];
        for (int k = 0; k < 3; k++) x[k] += t * V[k][e];
    }
    Mat N(3, 1, CV_32FC1);
    for (int k = 0; k < 3; k++) N.at<float>(k, 0) = (float)x[k];
    dst.assign(N);
    return true;
}
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
#define solve lexp_run_solve
#include "Utilities.hpp"
#include "Plane.h"
#include "StereoEnergy.h"
#include "Proposer.h"
#include "FastGCStereo.h"
#include "Evaluator.h"
#undef dilate
#undef solve
#include <omp.h>
#include <cstdio>
#include <stdexcept>

namespace {

struct RunProbe : FastGCStereo {
    using FastGCStereo::FastGCStereo;
    using FastGCStereo::selectRandomPixelInRect;
    using PMStereoBase::currentLabeling_;
    using PMStereoBase::currentLabeling_m_;
    using PMStereoBase::currentCost_;
    using PMStereoBase::stereoEnergy;
};
struct EvalProbe : Evaluator {
    using Evaluator::Evaluator;
    using Evaluator::validPixels;
    using Evaluator::nonoccPixels;
};

thread_local std::string g_err;

cv::Mat bgr(const uchar* p, int H, int W) { cv::Mat m(H, W, CV_8UC3); memcpy(m.data, p, (size_t)H * W * 3); return m; }
cv::Mat f32(const float* p, int H, int W) { cv::Mat m(H, W, CV_32F); memcpy(m.data, p, (size_t)H * W * 4); return m; }
cv::Mat u8(const uchar* p, int H, int W) { cv::Mat m(H, W, CV_8U); memcpy(m.data, p, (size_t)H * W); return m; }

// main.cpp:73 paramsGF with windR / lambda of the Options
Parameters params(int windR, float lambda) { Parameters p(1.0f, 20, "GF", 0.0001f); p.windR = windR; p.lambda = lambda; return p; }

// the last line of the Evaluator's log: Time, Eng, Data, Smooth, all, nonocc
int last_log_line(const std::string& path, double* out6) {
    FILE* f = fopen(path.c_str(), "r");
    if (!f) return -1;
    char line[1024];
    int ok = -1;
    while (fgets(line, sizeof line, f))
        if (sscanf(line, "%lf %lf %lf %lf %lf %lf", out6, out6 + 1, out6 + 2, out6 + 3, out6 + 4, out6 + 5) == 6) ok = 0;
    fclose(f);
    return ok;
}

}  // namespace

extern "C" {

const char* ref_run_last_error() { return g_err.c_str(); }

// initCurrentFast's random start (FastGCStereo.h:100-114) for n units: cv::theRNG().state = states[i], then
// selectRandomPixelInRect(unit i) and stereoEnergy->createRandomLabel(pixel) of an optimiser of the images (MIN 0, MAX max_disp).
int ref_run_random_start(int H, int W, const uchar* imL, const uchar* imR, float max_disp, int n, const int* units, const uint64_t* states,
                         float* out) {
    try {
        RunProbe s(bgr(imL, H, W), bgr(imR, H, W), params(20, 1.0f), max_disp, 0, 0);
        for (int i = 0; i < n; i++) {
            cv::theRNG().state = states[i];
            cv::Point p = s.selectRandomPixelInRect(cv::Rect(units[4 * i], units[4 * i + 1], units[4 * i + 2], units[4 * i + 3]));
            Plane l = s.stereoEnergy->createRandomLabel(p);
            out[4 * i] = l.a; out[4 * i + 1] = l.b; out[4 * i + 2] = l.c; out[4 * i + 3] = l.v;
        }
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// Evaluator(dispGT, nonocc, 255 / max_disp, .., log_dir)::evaluate(labeling_m, cost, energy, .., mode 0) with setPrecision(precision) and
// setErrorThreshold(threshold), on the given labeling [H][W][4] and cost [H][W].  nonocc: the mask as loadData leaves it (0 / 255).
// out: valid pixels, nonocc pixels, lastAccuracy (= all, full precision), then the log line's Time, Eng, Data, Smooth, all, nonocc.
int ref_run_evaluate(int H, int W, const uchar* imL, const uchar* imR, float max_disp, const float* labeling, const float* cost, const float* gt,
                     const uchar* nonocc, float precision, float threshold, const char* log_dir, double* out) {
    try {
        RunProbe s(bgr(imL, H, W), bgr(imR, H, W), params(20, 1.0f), max_disp, 0, 0);
        cv::Mat(H, W, CV_32FC4, (void*)labeling).copyTo(s.currentLabeling_[0]);
        f32(cost, H, W).copyTo(s.currentCost_[0]);
        EvalProbe ev(f32(gt, H, W), u8(nonocc, H, W), 255.0f / max_disp, "result", log_dir, false, false, true);
        ev.setPrecision(precision);
        ev.setErrorThreshold(threshold);
        ev.evaluate(s.currentLabeling_m_[0], s.currentCost_[0], *s.stereoEnergy, false, true, false, 0, 0);
        out[0] = ev.validPixels; out[1] = ev.nonoccPixels; out[2] = ev.lastAccuracy;
        return last_log_line(std::string(log_dir) + "log_output.txt", out + 3);
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// MidV2 of main.cpp:270-330 on the given pair: Evaluator with gt_prec and threshold 0.5, FastGCStereo with the layers 5 / 15 / 25 and
// main.cpp's proposer lists, cv::theRNG() of OpenMP thread j seeded with seed + j (main.cpp:443-450), run(iterations, {0, 1} or {0},
// pmIterations).  The accuracy of every evaluation of view 0 goes to log_dir/log_output.txt; out6 = its last line.
int ref_run_midv2(int H, int W, const uchar* imL, const uchar* imR, const float* gt, const uchar* nonocc, int ndisp, float gt_prec, int windR,
                  float lambda, int iterations, int pm_iterations, int do_dual, unsigned seed, const char* log_dir, double* out6) {
    try {
        const float maxdisp = (float)ndisp - 1;
        int nThread = omp_get_max_threads();
        #pragma omp parallel for
        for (int j = 0; j < nThread; j++) { srand(seed + j); cv::theRNG() = cv::RNG(seed + j); }
        Evaluator* eval = new Evaluator(f32(gt, H, W), u8(nonocc, H, W), 255.0f / maxdisp, "result", log_dir);
        eval->setPrecision(gt_prec);
        eval->showProgress = false;
        eval->setErrorThreshold(0.5f);
        {
            FastGCStereo stereo(bgr(imL, H, W), bgr(imR, H, W), params(windR, lambda), maxdisp, 0, 0);
            stereo.saveDir = log_dir;
            stereo.setEvaluator(eval);
            IProposer* prop1 = new ExpansionProposer(1);
            IProposer* prop2 = new RandomProposer(7, maxdisp);
            IProposer* prop3 = new ExpansionProposer(2);
            IProposer* prop4 = new RansacProposer(1);
            stereo.addLayer(5, {prop1, prop4, prop2});
            stereo.addLayer(15, {prop3, prop4});
            stereo.addLayer(25, {prop3, prop4});
            cv::Mat labeling, rawdisp;
            if (do_dual) stereo.run(iterations, {0, 1}, pm_iterations, labeling, rawdisp);
            else stereo.run(iterations, {0}, pm_iterations, labeling, rawdisp);
            delete prop1; delete prop2; delete prop3; delete prop4;
        }
        delete eval;   // closes the log
        return last_log_line(std::string(log_dir) + "log_output.txt", out6);
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

}  // extern "C"
