// TEST INFRASTRUCTURE ONLY -- never part of the product path.
//
// C entry points around the reference's OWN energies with a filterName of the caller's choice: CostVolumeEnergy with "BL"
// (BilateralFilter) or "" (no filter), NaiveStereoEnergy with "BF" or "" (CostVolumeEnergy.h:23-42, StereoEnergy.h:666-686),
// compiled from the reference's headers where they lie over the mini cv:: layer of oracle/cvshim/ (see oracle/build_ref_filters.py).
// Nothing here restates the algorithm: every cost returned is produced by ComputeUnaryPotential[WithoutCheck] and
// BilateralFilter::filter themselves.  Output: oracle/_ref/liblexp_ref_filters.so, which pins oracle/filter_oracle.py.
#include <opencv2/opencv.hpp>
#include "Utilities.hpp"
#include "Plane.h"
#include "StereoEnergy.h"
#include "CostVolumeEnergy.h"
#include <memory>
#include <string>

namespace {
thread_local std::string g_err;
struct ref_filter_ctx {
    std::unique_ptr<StereoEnergy> energy;
    cv::Mat im[2];
};
}  // namespace

extern "C" {

const char* ref_filter_last_error() { return g_err.c_str(); }

// kind 0: CostVolumeEnergy (volumes [D][H][W] float, borrowed: the caller keeps them alive); kind 1: NaiveStereoEnergy.  Images 8-bit
// BGR [H][W][3]; filter_name as Parameters::filterName; param1 = Parameters::filter_param1 (sig2 of the bilateral filter).
void* ref_filter_create(int kind, int H, int W, int D, const uchar* imL, const uchar* imR, float* volL, float* volR, int windR,
                        const char* filter_name, float param1, float th_col, float th_grad, float alpha, float max_disp, float min_disp) {
    try {
        auto c = std::make_unique<ref_filter_ctx>();
        c->im[0] = cv::Mat(H, W, CV_8UC3, (void*)imL).clone();
        c->im[1] = cv::Mat(H, W, CV_8UC3, (void*)imR).clone();
        Parameters params(20.f, windR, filter_name, param1);
        params.th_col = th_col; params.th_grad = th_grad; params.alpha = alpha;
        if (kind == 0) {
            int sz[3] = {D, H, W};
            cv::Mat vL(3, sz, CV_32F, volL), vR(3, sz, CV_32F, volR);
            c->energy = std::make_unique<CostVolumeEnergy>(c->im[0], c->im[1], vL, vR, params, max_disp, min_disp);
        } else {
            c->energy = std::make_unique<NaiveStereoEnergy>(c->im[0], c->im[1], params, max_disp, min_disp);
        }
        return c.release();
    } catch (const std::exception& e) { g_err = e.what(); return nullptr; }
}
void ref_filter_destroy(void* h) { delete (ref_filter_ctx*)h; }

// One call of the virtual as FastGCStereo.h:47 issues it: `out` is the filterRect-sized view proposalCost(filterRect) ([fh][fw] float,
// caller-initialised; only the target sub-rectangle is written).
int ref_filter_unary(void* h, const int frect[4], const int trect[4], const float plane[4], int mode, int with_check, float* out) {
    try {
        ref_filter_ctx* c = (ref_filter_ctx*)h;
        cv::Rect fr(frect[0], frect[1], frect[2], frect[3]), tr(trect[0], trect[1], trect[2], trect[3]);
        cv::Mat costs(fr.height, fr.width, CV_32F, out);
        Plane p(plane[0], plane[1], plane[2], plane[3]);
        StereoEnergy::Reusable reusable;
        if (with_check) c->energy->ComputeUnaryPotential(fr, tr, costs, p, reusable, mode);
        else c->energy->ComputeUnaryPotentialWithoutCheck(fr, tr, costs, p, reusable, mode);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return 1; }
}

}  // extern "C"
