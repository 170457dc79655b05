// lexp_vis.cuh -- the reference's debug images on the device (DESIGN.md section 3j): what Evaluator::evaluate writes at every
// evaluation point (Evaluator.h:123-166, resultmD / resultmN / resultmE) and the images of viewConsistencyCheck (PMStereoBase.h:87-108,
// result0C / result1C).  Every image is 8-bit, row-major, channel-interleaved BGR where it has three channels.
//
//   lexp_vis_eval_kernel    one view, one thread per pixel:
//     D = sat8((float)((float)disp * alpha) * 255.0f)              alpha = (float)((double)(255.0f / max_disp) * (1.0 / 255)): OpenCV folds
//                                                                  disp * F / 255 into one float convertTo; * 255 is the second one
//     N = sat8(255.0f * (nz, (-b nz + 1) / 2, (-a nz + 1) / 2))    nz = 1 / sqrt(a a + b b + 1), every operation rounded to float
//     E = 255 where ok or GT is invalid, else 200 where occluded (valid GT, nonocc == 0), else 0
//   disp, its quantisation and ok are eval_pixel's (lexp_run.cuh), the arithmetic of lexp_evaluate; view 1 is scored against the left GT.
//   lexp_vis_check_kernel   both views, one thread per pixel, from the fail map of lexp_post_check_kernel (threshold 1.5):
//     gray = sat8((float)disp * s + o), s = 255.0f / (max_disp - min_disp), o = -min_disp * s
//     BGR  = (fail == 128 ? 255 : gray, gray, fail == 255 ? 255 : gray)
// sat8 = saturate_cast<uchar>(float): cvRound (round half to even; NaN and values outside int32 give INT_MIN), then clamp to 0 .. 255.
//
// The kernels live in lexp_vis.cu, built into their own library (liblexp_vis.so, which liblexp_cuda.so links): liblexp_cuda.so carries
// exactly the kernels it carried before.  This header declares their launchers.  Neither kernel writes any state of the context.
#pragma once
#include "lexp_run.cuh"

#define LEXP_VIS_API __attribute__((visibility("default")))

namespace lexp {

constexpr int kVisThreads = 256;

// Launchers on `stream` (lexp_vis.cu).  Any of d, n_bgr, e may be null: that image is not written.
LEXP_VIS_API cudaError_t vis_launch_eval(const float4* cur_label, const float* gt, const unsigned char* nonocc, unsigned char* d, unsigned char* n_bgr,
                                         unsigned char* e, int H, int W, float precision, float threshold, float max_disp, cudaStream_t stream);
// fail: [2][H][W] of lexp_post_check_kernel; c_bgr: [2][H][W][3]
LEXP_VIS_API cudaError_t vis_launch_check(const float4* lab0, const float4* lab1, const unsigned char* fail, unsigned char* c_bgr, int H, int W,
                                          float min_disp, float max_disp, cudaStream_t stream);

}  // namespace lexp
