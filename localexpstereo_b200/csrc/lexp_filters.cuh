// lexp_filters.cuh -- the reference's other two aggregation filters on the device: the bilateral filter (filterName "BL" for
// CostVolumeEnergy, "BF" for NaiveStereoEnergy) and no filter at all ("").  The contract is DESIGN.md section 3i.
//
//   "":        q(x) = p(x), the raw cost itself (CostVolumeEnergy.h:169-171, StereoEnergy.h:752-753).
//   bilateral: q(x) = sum over y in (x +- windR) & filterRect of p(y) exp(-(|I0(y)-I0(x)| + |I1(y)-I1(x)| + |I2(y)-I2(x)|) / sig2)
//              (GuidedFilter.h:329-373): radius windR (not the guided filter's windR / 2), guide = the 8-bit BGR image unscaled, the
//              window clipped at the filterRect (createSubregionFilter gives I(rect) its own domain), the sum not normalised.
//
// Raw costs come from the samplers of lexp_label_cost.cuh (team A's arithmetic of lexp_fused_kernel, every operation rounded
// separately) and, for NaiveStereoEnergy, the call's inverse affine map naive_inverse_affine: bit-identical raw costs.  The channel
// sum of a weight is an integer in [0, 765], so the weights come from a table exp(-s / sig2) computed once per context in FP64 and
// rounded to float (correctly rounded weights, no MUFU in the inner loop).  Every output sums its window in one fixed order --
// row by row from the top, each row from the left into its own partial sum with fmaf, the row sums added in order -- so two calls
// give the same bits, and a 1x1 call on F(p) gives the same bits as the warm-start kernel for p.
//
// The kernels live in lexp_filters.cu, built into their own library (liblexp_filters.so, which liblexp_cuda.so links): liblexp_cuda.so
// carries exactly the kernels it carried before.  This header declares their launchers.
// Kernels (ordinary stream-ordered launches, no programmatic-dependent-launch attribute):
//   lexp_filter_unary_kernel<NAIVE, FILTER>    the unary calls of a plan, one CTA per planner work item (run_plan's outputs)
//   lexp_filter_label_cost_kernel<NAIVE, FILTER>  initCurrentFast from a labeling (DESIGN.md 3g), one CTA per pixel
//   lexp_filter_pm_update_kernel                the PatchMatch update of a step over the group's targetRects
#pragma once
#include "lexp_kernels.cuh"
#include "lexp_gc.cuh"
#include "lexp_label_cost.cuh"

#define LEXP_FILTERS_API __attribute__((visibility("default")))

namespace lexp {

constexpr int kFtThreads = 256;
constexpr int kFtBW = 32, kFtBH = 8;   // output sub-tile of one pass of lexp_filter_unary_kernel: one thread per pixel
constexpr int kFtWsThreads = 128;      // lexp_filter_label_cost_kernel: one thread per window row (2 windR + 1 <= 99)
constexpr int kBlWeights = 766;        // channel sums 0 .. 3 * 255

struct FtParams {
    LcParams lc;                          // the samplers' inputs (volume, ExI, guide, sizes, thresholds, view)
    const Item* __restrict__ items;
    const Plane4* __restrict__ planes;
    float* __restrict__ out;
    long long out_pitch;                  // floats per row (image mode)
    int out_compact;                      // 1: per-call contiguous tiles, 0: H x W image
    int with_check;
    const float* __restrict__ wtab;       // [kBlWeights] exp(-s / sig2) (bilateral only)
};

// dynamic shared memory of lexp_filter_unary_kernel: weights, inverse affine map, raw costs and guide of the staged region
// (sub-tile +- windR), the naive warp's fixed-point row terms and column deltas
__host__ __device__ inline size_t filter_unary_smem_bytes(int windR, bool bilateral) {
    const int wR = bilateral ? windR : 0;
    const size_t SR = kFtBH + 2 * wR, SC = kFtBW + 2 * wR;
    return 6 * 8 + (size_t)kBlWeights * 4 + SR * SC * 8 + 2 * SR * 4 + 2 * SC * 4;
}

// Launchers on `stream` (lexp_filters.cu).  `configured`: the kernel's dynamic shared-memory opt-in up to smem_limit has been made.
LEXP_FILTERS_API cudaError_t filter_launch_unary(bool naive, bool bilateral, const FtParams& p, unsigned nitems, size_t smem, size_t smem_limit,
                                                 bool& configured, cudaStream_t stream);
LEXP_FILTERS_API cudaError_t filter_launch_label_cost(bool naive, bool bilateral, const LcParams& p, const float* wtab, cudaStream_t stream);
LEXP_FILTERS_API cudaError_t filter_launch_pm_update(unsigned ncalls, const GcCell* cells, const Plane4* planes, const float* prop_cost, float* cur_cost,
                                                     float4* cur_label, int W, int init, int* flags, const int* epoch_base, int rank,
                                                     int publish_epoch, cudaStream_t stream);

}  // namespace lexp
