// lexp_vis.cu -- the kernels of lexp_vis.cuh (the reference's debug images, DESIGN.md 3j) and their launchers.
// Built into liblexp_vis.so by localexpstereo_b200/build.py; the CPU emulator of tests/emu compiles it into its one translation unit
// (lexp_capi.cu includes it under LEXP_EMU).  As with lexp_filters.cu, the headers it includes make this library compile copies of the
// non-template kernels they define; nothing launches those copies.
#include "../../include/lexp_cuda.h"
#include "lexp_vis.cuh"

#ifndef LEXP_EMU
#define LEXP_VIS_LAUNCH(kern, grid, block, stream, ...) kern<<<grid, block, 0, stream>>>(__VA_ARGS__)
#else
#define LEXP_VIS_LAUNCH(kern, grid, block, stream, ...) emu::launch(kern, dim3(grid), dim3(block), (size_t)0, __VA_ARGS__)
#endif

namespace lexp {

// saturate_cast<uchar>(float) as OpenCV computes it on x86-64: cvRound (cvtss2si: round half to even, INT_MIN for NaN and for values
// outside int32), then clamp to 0 .. 255
__device__ __forceinline__ unsigned char vis_sat8(float v) {
    if (!(v >= -2147483648.0f && v < 2147483648.0f)) return 0;
#ifndef LEXP_EMU
    const int r = __float2int_rn(v);
#else
    const int r = (int)nearbyintf(v);
#endif
    return (unsigned char)(r < 0 ? 0 : r > 255 ? 255 : r);
}

__device__ __forceinline__ float vis_sqrt(float v) {
#ifndef LEXP_EMU
    return __fsqrt_rn(v);
#else
    volatile float r = sqrtf(v);
    return r;
#endif
}

__global__ void __launch_bounds__(kVisThreads) lexp_vis_eval_kernel(const float4* __restrict__ cur_label, const float* __restrict__ gt,
                                                                    const unsigned char* __restrict__ nonocc, unsigned char* __restrict__ d_out,
                                                                    unsigned char* __restrict__ n_out, unsigned char* __restrict__ e_out, int H, int W,
                                                                    float precision, float threshold, float alpha) {
    const long long p = (long long)blockIdx.x * kVisThreads + threadIdx.x;
    if (p >= (long long)H * W) return;
    const int x = (int)(p % W), y = (int)(p / W);
    const float4 L = cur_label[p];
    const float g = gt[p];
    int valid = 0, ok = 0;
    const float d = eval_pixel(L, g, x, y, precision, threshold, valid, ok);
    if (d_out) d_out[p] = vis_sat8(__fmul_rn(__fadd_rn(__fmul_rn(d, alpha), 0.0f), 255.0f));   // (disp * F / 255) * 255
    if (n_out) {   // StereoEnergy::computeNormalMap (StereoEnergy.h:274-289), then * 255
        const float nz = __fdiv_rn(1.0f, vis_sqrt(__fadd_rn(__fadd_rn(__fmul_rn(L.x, L.x), __fmul_rn(L.y, L.y)), 1.0f)));
        const float gch = __fmul_rn(__fadd_rn(-__fmul_rn(L.y, nz), 1.0f), 0.5f);
        const float rch = __fmul_rn(__fadd_rn(-__fmul_rn(L.x, nz), 1.0f), 0.5f);
        unsigned char* o = n_out + 3 * p;
        o[0] = vis_sat8(__fmul_rn(nz, 255.0f));
        o[1] = vis_sat8(__fmul_rn(gch, 255.0f));
        o[2] = vis_sat8(__fmul_rn(rch, 255.0f));
    }
    if (e_out) e_out[p] = (ok || !valid) ? 255 : (nonocc[p] ? 0 : 200);   // errorMap | ~validMask; 200 on occMask & ~errorMapVis
}

__global__ void __launch_bounds__(kVisThreads) lexp_vis_check_kernel(const float4* __restrict__ lab0, const float4* __restrict__ lab1,
                                                                     const unsigned char* __restrict__ fail, unsigned char* __restrict__ c_out, int H, int W,
                                                                     float s, float o) {
    const long long HW = (long long)H * W;
    const long long p = (long long)blockIdx.x * kVisThreads + threadIdx.x;
    const int m = blockIdx.y;
    if (p >= HW) return;
    const int x = (int)(p % W), y = (int)(p / W);
    const float d = gc_disp((m ? lab1 : lab0)[p], (float)x, (float)y);   // computeDisparities(currentLabeling_[m])
    const unsigned char gray = vis_sat8(__fadd_rn(__fmul_rn(d, s), o));     // convertTo(CV_8U, dispVisScaling, dispVisOffset)
    const unsigned char f = fail[m * HW + p];
    unsigned char* out = c_out + 3 * (m * HW + p);
    out[0] = f == 128 ? 255 : gray;
    out[1] = gray;
    out[2] = f == 255 ? 255 : gray;
}

cudaError_t vis_launch_eval(const float4* cur_label, const float* gt, const unsigned char* nonocc, unsigned char* d, unsigned char* n_bgr, unsigned char* e,
                            int H, int W, float precision, float threshold, float max_disp, cudaStream_t stream) {
    // DISPARITY_FACTOR = 255.0f / maxdisp (main.cpp:291,380); disp * F / 255 is one convertTo with scale (double)F * (1.0 / 255)
    const float alpha = (float)((double)(255.0f / max_disp) * (1.0 / 255));
    const unsigned nblocks = (unsigned)(((long long)H * W + kVisThreads - 1) / kVisThreads);
    LEXP_VIS_LAUNCH(lexp_vis_eval_kernel, nblocks, kVisThreads, stream, cur_label, gt, nonocc, d, n_bgr, e, H, W, precision, threshold, alpha);
    return cudaGetLastError();
}

cudaError_t vis_launch_check(const float4* lab0, const float4* lab1, const unsigned char* fail, unsigned char* c_bgr, int H, int W, float min_disp,
                             float max_disp, cudaStream_t stream) {
    const float s = 255.0f / (max_disp - min_disp);   // dispVisScaling, dispVisOffset (PMStereoBase.h:51-52), float arithmetic
    const float o = -min_disp * s;
    const unsigned nblocks = (unsigned)(((long long)H * W + kVisThreads - 1) / kVisThreads);
    LEXP_VIS_LAUNCH(lexp_vis_check_kernel, dim3(nblocks, 2), kVisThreads, stream, lab0, lab1, fail, c_bgr, H, W, s, o);
    return cudaGetLastError();
}

}  // namespace lexp
