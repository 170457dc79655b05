// lexp_run.cuh -- the two pieces of FastGCStereo::run that have no other kernel: the random start of initCurrentFast and the Evaluator.
//
//   lexp_random_start_kernel   initCurrentFast with an empty labeling (FastGCStereo.h:100-114): one label per layer-0 unit,
//                              selectRandomPixelInRect (FastGCStereo.h:229-236) + StereoEnergy::createRandomLabel (StereoEnergy.h:120-129)
//                              from CvRng{pm_rng_state(seed, cell_id)}, MAX_VDISPARITY = 0.  Restated by oracle.run_oracle.random_start.
//   lexp_eval_kernel /         Evaluator::evaluate (Evaluator.h:113-187): the disparity of every pixel (computeDisparities, gc_disp), its
//   lexp_eval_finish           quantisation (convertTo CV_32S with 1 / precision, then back), |disp - GT| <= threshold, and the four pixel
//                              counts of the `all` / `nonocc` rates.  Integer counts per block, added up in block order: the same result on
//                              every call.
#pragma once
#include <climits>
#include "lexp_kernels.cuh"
#include "lexp_gc.cuh"

namespace lexp {

// One thread per unit: the label the unit starts from (one per call of the plan, written into `planes`, which the init step then reads like
// a list).  Every floating-point operation rounded as the reference's host code (as in pm_propose).
__global__ void lexp_random_start_kernel(const CallInfo* __restrict__ calls, int n, Plane4* __restrict__ planes, unsigned long long seed,
                                         float min_disp, float max_disp) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const CallInfo ci = calls[i];
    CvRng rng{pm_rng_state(seed, ci.cell_id)};
    const int k = rng.uniform_int(0, ci.uw * ci.uh);                                    // selectRandomPixelInRect
    const float fx = (float)(ci.ux + k % ci.uw), fy = (float)(ci.uy + k / ci.uw);
    const float zs = rng.uniform_float(min_disp, max_disp);                             // createRandomLabel
    const double theta = rng.uniform_double(0.0, __ddiv_rn(3.14159265358979323846, 3.0));   // getRandomUnitVector(CV_PI / 3)
    const double phi = rng.uniform_double(0.0, __dmul_rn(3.14159265358979323846, 2.0));
    const double cT = cos(theta), sT = sin(theta), cP = cos(phi), sP = sin(phi);
    const float nx = (float)__dmul_rn(sT, cP), ny = (float)__dmul_rn(sT, sP), nz = (float)cT;   // Vec3d -> Vec<float, 3>
    Plane4 out;                                                                         // Plane::CreatePlane (Plane.h:23-31)
    out.a = __fdiv_rn(-nx, nz);
    out.b = __fdiv_rn(-ny, nz);
    out.c = __fsub_rn(__fsub_rn(zs, __fmul_rn(out.a, fx)), __fmul_rn(out.b, fy));
    out.v = 0.0f;
    planes[i] = out;
}

constexpr int kEvalThreads = 256;

// cvRound of a double as the x86 conversion does it (round half to even; NaN and results outside int32 give INT_MIN)
__device__ __forceinline__ int eval_cvround(double s) {
    return (s >= -2147483648.5 && s < 2147483647.5) ? __double2int_rn(s) : INT_MIN;
}

// The Evaluator's arithmetic at one pixel (Evaluator.h:123-139), shared by lexp_eval_kernel and the debug images of lexp_vis.cuh:
// the disparity of `label` at (x, y), quantised when precision > 0 (returned in d), whether GT g is valid, and errorMap's predicate.
__device__ __forceinline__ float eval_pixel(const float4 label, float g, int x, int y, float precision, float threshold, int& valid, int& ok) {
    float d = gc_disp(label, (float)x, (float)y);
    if (precision > 0.0f) {   // quantize (Evaluator.h:105-110): m.convertTo(CV_32S, 1.0 / precision), then back with scale precision
        // cvtScale 32f -> 32s works in float: (float)src * (float)alpha + (float)beta, then cvRound; 32s -> 32f works in double
        const float s = __fadd_rn(__fmul_rn(d, (float)__ddiv_rn(1.0, (double)precision)), 0.0f);
        const int q = eval_cvround((double)s);
        d = (float)__dmul_rn((double)q, (double)precision);
    }
    valid = (g > 0.0f && g <= 3.402823466e+38f) ? 1 : 0;   // validMask = GT > 0 & GT != inf
    ok = ((double)fabsf(__fsub_rn(d, g)) <= (double)threshold) ? 1 : 0;   // errorMap = |disp - GT| <= errorThreshold
    return d;
}

// part[4 b + k], k = valid pixels, nonocc pixels, correct & valid, correct & nonocc of block b
__global__ void __launch_bounds__(kEvalThreads) lexp_eval_kernel(const float4* __restrict__ cur_label, const float* __restrict__ gt,
                                                                 const unsigned char* __restrict__ nonocc, long long* __restrict__ part, int H, int W,
                                                                 float precision, float threshold) {
    __shared__ unsigned char s_bits[kEvalThreads];
    const long long p = (long long)blockIdx.x * kEvalThreads + threadIdx.x;
    int valid = 0, nocc = 0, ok = 0;
    if (p < (long long)H * W) {
        const int x = (int)(p % W), y = (int)(p / W);
        eval_pixel(cur_label[p], gt[p], x, y, precision, threshold, valid, ok);
        nocc = nonocc[p] ? 1 : 0;
    }
    s_bits[threadIdx.x] = (unsigned char)(valid | nocc << 1 | (ok & valid) << 2 | (ok & nocc) << 3);
    __syncthreads();
    if (threadIdx.x == 0) {
        long long c[4] = {0, 0, 0, 0};
        for (int t = 0; t < kEvalThreads; t++)
            for (int k = 0; k < 4; k++) c[k] += (s_bits[t] >> k) & 1;
        long long* o = part + 4 * (size_t)blockIdx.x;
        for (int k = 0; k < 4; k++) o[k] = c[k];
    }
}
// thread k < 4 adds up count k of every block (integers: the order does not change the sum)
__global__ void lexp_eval_finish(const long long* __restrict__ part, int nblocks, long long* __restrict__ out4) {
    const int k = threadIdx.x;
    if (k >= 4) return;
    long long s = 0;
    for (int b = 0; b < nblocks; b++) s += part[4 * (size_t)b + k];
    out4[k] = s;
}

}  // namespace lexp
