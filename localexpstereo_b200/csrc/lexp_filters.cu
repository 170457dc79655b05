// lexp_filters.cu -- the kernels of lexp_filters.cuh (the bilateral filter and the unfiltered mode, DESIGN.md 3i) and their launchers.
// Built into liblexp_filters.so by localexpstereo_b200/build.py; the CPU emulator of tests/emu compiles it into its one translation
// unit (lexp_capi.cu includes it under LEXP_EMU).
// lexp_filters.cuh includes lexp_kernels.cuh (Item, Plane4, naive_inverse_affine) and lexp_gc.cuh (GcCell), so this library also compiles
// the non-template kernels those headers define (the graph-cut, energy and statistics kernels).  Nothing launches those copies: the
// launchers below name only the kernels of this file, and the host stubs stay private to each library (-fvisibility=hidden).  Moving the
// shared types into headers of their own would change the headers liblexp_cuda.so is built from.
#include "../../include/lexp_cuda.h"
#include "lexp_filters.cuh"

#ifndef LEXP_EMU
#define LEXP_FT_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<grid, block, smem, stream>>>(__VA_ARGS__)
#else
#define LEXP_FT_LAUNCH(kern, grid, block, smem, stream, ...) emu::launch(kern, dim3(grid), dim3(block), (size_t)(smem), __VA_ARGS__)
#endif

namespace lexp {

// channel sum of |a - b| over the three guide bytes (the fourth byte is 0 in both)
__device__ __forceinline__ int bl_sad(unsigned a, unsigned b) {
#ifndef LEXP_EMU
    return (int)__vsadu4(a, b);
#else
    int s = 0;
    for (int k = 0; k < 32; k += 8) s += abs((int)((a >> k) & 255u) - (int)((b >> k) & 255u));
    return s;
#endif
}

// IsValiLabel (StereoEnergy.h:560-610) at (x, y), as team E of lexp_fused_kernel evaluates it: the plane at p and at p +- (5, 5)
// inside [MIN, MAX]; a targetRect larger than 1x1 adds channelSum's 4th term 0 * v
__device__ __forceinline__ bool ft_valid(const Plane4 pl, int x, int y, bool one_by_one, float lo, float hi) {
    float ds = __fadd_rn(__fadd_rn(__fmul_rn((float)x, pl.a), __fmul_rn((float)y, pl.b)), pl.c);
    if (!one_by_one) ds = __fadd_rn(ds, __fmul_rn(0.0f, pl.v));
    const float a5 = __fmul_rn(pl.a, 5.0f), b5 = __fmul_rn(pl.b, 5.0f);
    const float dpp = __fadd_rn(__fadd_rn(ds, a5), b5), dpm = __fsub_rn(__fadd_rn(ds, a5), b5);
    const float dmp = __fadd_rn(__fsub_rn(ds, a5), b5), dmm = __fsub_rn(__fsub_rn(ds, a5), b5);
    return ds >= lo && ds <= hi && dpp >= lo && dpp <= hi && dpm >= lo && dpm <= hi && dmp >= lo && dmp <= hi && dmm >= lo && dmm <= hi;
}

// cv::warpAffine fixed-point row term / column delta (AB_BITS = 10, round_delta = 16) of a row / column relative to the filterRect
__device__ __forceinline__ void ft_row_terms(const double* iM, int yr, int& rx, int& ry) {
    rx = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(iM[1], (double)yr), iM[2]), 1024.0)) + 16;
    ry = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(iM[4], (double)yr), iM[5]), 1024.0)) + 16;
}
__device__ __forceinline__ void ft_col_terms(const double* iM, int xr, int& ca, int& cb) {
    ca = __double2int_rn(__dmul_rn(__dmul_rn(iM[0], (double)xr), 1024.0));
    cb = __double2int_rn(__dmul_rn(__dmul_rn(iM[3], (double)xr), 1024.0));
}

// grid = plan items; block = kFtThreads.  FILTER: LEXP_FILTER_BILATERAL or LEXP_FILTER_NONE.
template <bool NAIVE, int FILTER>
__global__ void __launch_bounds__(kFtThreads) lexp_filter_unary_kernel(const FtParams P) {
    constexpr bool BL = FILTER == LEXP_FILTER_BILATERAL;
    const Item it = P.items[blockIdx.x];
    const Plane4 pl = P.planes[it.call];
    const int tid = threadIdx.x;
    const int wR = BL ? P.lc.windR : 0;
    const int SR = kFtBH + 2 * wR, SC = kFtBW + 2 * wR;
    const int fx1 = it.fx + it.fw, fy1 = it.fy + it.fh;
    const int W = P.lc.W;
    LEXP_DYNAMIC_SMEM(smem_raw);
    double* s_iM = reinterpret_cast<double*>(smem_raw);            // [6]
    float* s_w = reinterpret_cast<float*>(s_iM + 6);               // [kBlWeights]
    float* s_p = s_w + kBlWeights;                                  // [SR][SC] raw costs of the staged region
    unsigned* s_g = reinterpret_cast<unsigned*>(s_p + SR * SC);     // [SR][SC] guide (BGR0 bytes)
    int* s_rx = reinterpret_cast<int*>(s_g + SR * SC);              // NAIVE [SR] x 2, [SC] x 2
    int* s_ry = s_rx + SR;
    int* s_ca = s_ry + SR;
    int* s_cb = s_ca + SC;
    if (NAIVE && tid == 0) naive_inverse_affine(it, pl, P.lc.mode, s_iM);
    if (BL)
        for (int i = tid; i < kBlWeights; i += kFtThreads) s_w[i] = P.wtab[i];
    __syncthreads();

    const int tx = tid % kFtBW, ty = tid / kFtBW;
    for (int sy0 = it.oy0; sy0 < it.oy0 + it.oh; sy0 += kFtBH)
        for (int sx0 = it.ox0; sx0 < it.ox0 + it.ow; sx0 += kFtBW) {
            // staged region: (sub-tile +- windR) & filterRect
            const int ry0 = max(sy0 - wR, it.fy), ry1 = min(sy0 + kFtBH + wR, fy1);
            const int rx0 = max(sx0 - wR, it.fx), rx1 = min(sx0 + kFtBW + wR, fx1);
            const int nr = ry1 - ry0, nc = rx1 - rx0;
            if (NAIVE) {
                for (int j = tid; j < nr; j += kFtThreads) ft_row_terms(s_iM, ry0 + j - it.fy, s_rx[j], s_ry[j]);
                for (int i = tid; i < nc; i += kFtThreads) ft_col_terms(s_iM, rx0 + i - it.fx, s_ca[i], s_cb[i]);
                __syncthreads();
            }
            for (int k = tid; k < nr * nc; k += kFtThreads) {
                const int j = k / nc, i = k - j * nc;
                const int y = ry0 + j, x = rx0 + i;
                s_p[k] = NAIVE ? lc_raw_naive(P.lc, x, y, s_rx[j] + s_ca[i], s_ry[j] + s_cb[i]) : lc_raw_volume(P.lc, pl, x, y);
                if (BL) s_g[k] = __ldg(reinterpret_cast<const unsigned*>(P.lc.guide) + (size_t)y * W + x);
            }
            __syncthreads();
            const int x = sx0 + tx, y = sy0 + ty;
            if (x < it.ox0 + it.ow && y < it.oy0 + it.oh) {
                const int c = (y - ry0) * nc + (x - rx0);
                float q = s_p[c];
                if (BL) {
                    const unsigned gc = s_g[c];
                    const int wy0 = max(y - wR, it.fy), wy1 = min(y + wR + 1, fy1);
                    const int wx0 = max(x - wR, it.fx) - rx0, wx1 = min(x + wR + 1, fx1) - rx0;
                    q = 0.0f;
                    for (int yy = wy0; yy < wy1; yy++) {
                        const float* pr = s_p + (yy - ry0) * nc;
                        const unsigned* gr = s_g + (yy - ry0) * nc;
                        float r = 0.0f;
                        for (int xx = wx0; xx < wx1; xx++) r = fmaf(pr[xx], s_w[bl_sad(gr[xx], gc)], r);
                        q = __fadd_rn(q, r);
                    }
                }
                if (P.with_check && !ft_valid(pl, x, y, (it.flags & 1) != 0, P.lc.min_disp, P.lc.max_disp)) q = kCostInvalid;   // :180-182
                float* o = P.out_compact ? P.out + (size_t)it.compact_off + (size_t)(y - it.oy0) * it.compact_stride + (x - it.ox0)
                                         : P.out + (size_t)y * P.out_pitch + x;
                *o = q;
            }
            __syncthreads();   // the next pass overwrites the staged region
        }
}

// initCurrentFast from the labeling the state holds (FastGCStereo.h:116-130) with the bilateral filter or none: for every pixel p,
// currentCost_(p) = ComputeUnaryPotential(F(p), {p}, ., currentLabeling_(p)), F(p) = (p +- windR) & image.  The bilateral window
// (p +- windR) & F(p) is F(p) itself.  grid = (W, H), block = kFtWsThreads: thread j sums row F.y + j of the window, thread 0 adds
// the row sums in order -- the same operations as lexp_filter_unary_kernel on the call (F(p), {p}).
template <bool NAIVE, int FILTER>
__global__ void __launch_bounds__(kFtWsThreads) lexp_filter_label_cost_kernel(const LcParams P, const float* __restrict__ wtab) {
    constexpr bool BL = FILTER == LEXP_FILTER_BILATERAL;
    __shared__ double s_iM[6];
    __shared__ float s_row[kFtWsThreads];
    const int px = blockIdx.x, py = blockIdx.y, tid = threadIdx.x;
    const int H = P.H, W = P.W, wR = P.windR;
    const size_t pix = (size_t)py * W + px;
    const float4 l4 = P.label[pix];
    const Plane4 pl{l4.x, l4.y, l4.z, l4.w};
    Item it{};   // F(p): the reference's filterRegion of a 1x1 unit
    it.fx = max(px - wR, 0); it.fy = max(py - wR, 0);
    it.fw = min(px + wR + 1, W) - it.fx; it.fh = min(py + wR + 1, H) - it.fy;
    if (NAIVE && tid == 0) naive_inverse_affine(it, pl, P.mode, s_iM);
    __syncthreads();
    auto raw = [&](int x, int y) {
        if (!NAIVE) return lc_raw_volume(P, pl, x, y);
        int rx, ry, ca, cb;
        ft_row_terms(s_iM, y - it.fy, rx, ry);
        ft_col_terms(s_iM, x - it.fx, ca, cb);
        return lc_raw_naive(P, x, y, rx + ca, ry + cb);
    };
    if (!BL) {
        if (tid == 0) {
            float q = raw(px, py);
            if (!ft_valid(pl, px, py, true, P.min_disp, P.max_disp)) q = kCostInvalid;
            P.cost[pix] = q;
        }
        return;
    }
    const unsigned* guide = reinterpret_cast<const unsigned*>(P.guide);
    const unsigned gc = __ldg(guide + pix);
    if (tid < it.fh) {
        const int y = it.fy + tid;
        float r = 0.0f;
        for (int x = it.fx; x < it.fx + it.fw; x++) r = fmaf(raw(x, y), __ldg(wtab + bl_sad(__ldg(guide + (size_t)y * W + x), gc)), r);
        s_row[tid] = r;
    }
    __syncthreads();
    if (tid == 0) {
        float q = 0.0f;
        for (int j = 0; j < it.fh; j++) q = __fadd_rn(q, s_row[j]);
        if (!ft_valid(pl, px, py, true, P.min_disp, P.max_disp)) q = kCostInvalid;
        P.cost[pix] = q;
    }
}

// The update of a decomposed PatchMatch step (FastGCStereo.h:56-60): after the unary costs of the proposals are in prop_cost, every
// pixel of every call's targetRect takes (q, proposal) where currentCost > q -- NaN never updates -- or unconditionally for an
// initialisation step (:105-113).  One CTA per call.  publish_epoch != 0 (last step of a group): flags[rank] = base + publish_epoch,
// as lexp_fused_kernel leaves it.
__global__ void lexp_filter_pm_update_kernel(const GcCell* __restrict__ cells, const Plane4* __restrict__ planes, const float* __restrict__ prop_cost,
                                             float* __restrict__ cur_cost, float4* __restrict__ cur_label, int W, int init,
                                             int* flags, const int* epoch_base, int rank, int publish_epoch) {
    const GcCell c = cells[blockIdx.x];
    const Plane4 pl = planes[blockIdx.x];
    const float4 l1 = make_float4(pl.a, pl.b, pl.c, pl.v);
    const int N = c.w * c.h;
    for (int s = threadIdx.x; s < N; s += blockDim.x) {
        const size_t p = (size_t)(c.y + s / c.w) * W + (c.x + s % c.w);
        const float q = prop_cost[p];
        if (init || cur_cost[p] > q) {
            cur_cost[p] = q;
            cur_label[p] = l1;
        }
    }
    if (publish_epoch && blockIdx.x == 0 && threadIdx.x == 0) flags[rank] = *epoch_base + publish_epoch;
}


cudaError_t filter_launch_unary(bool naive, bool bilateral, const FtParams& p, unsigned nitems, size_t smem, size_t smem_limit, bool& configured,
                                cudaStream_t stream) {
    auto kern = naive ? (bilateral ? lexp_filter_unary_kernel<true, LEXP_FILTER_BILATERAL> : lexp_filter_unary_kernel<true, LEXP_FILTER_NONE>)
                      : (bilateral ? lexp_filter_unary_kernel<false, LEXP_FILTER_BILATERAL> : lexp_filter_unary_kernel<false, LEXP_FILTER_NONE>);
    if (!configured) {
        const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit);
        if (e != cudaSuccess) return e;
        configured = true;
    }
    LEXP_FT_LAUNCH(kern, nitems, kFtThreads, smem, stream, p);
    return cudaGetLastError();
}

cudaError_t filter_launch_label_cost(bool naive, bool bilateral, const LcParams& p, const float* wtab, cudaStream_t stream) {
    auto kern = naive ? (bilateral ? lexp_filter_label_cost_kernel<true, LEXP_FILTER_BILATERAL> : lexp_filter_label_cost_kernel<true, LEXP_FILTER_NONE>)
                      : (bilateral ? lexp_filter_label_cost_kernel<false, LEXP_FILTER_BILATERAL> : lexp_filter_label_cost_kernel<false, LEXP_FILTER_NONE>);
    LEXP_FT_LAUNCH(kern, dim3((unsigned)p.W, (unsigned)p.H), kFtWsThreads, 0, stream, p, wtab);
    return cudaGetLastError();
}

cudaError_t filter_launch_pm_update(unsigned ncalls, const GcCell* cells, const Plane4* planes, const float* prop_cost, float* cur_cost,
                                    float4* cur_label, int W, int init, int* flags, const int* epoch_base, int rank, int publish_epoch,
                                    cudaStream_t stream) {
    LEXP_FT_LAUNCH(lexp_filter_pm_update_kernel, ncalls, 256, 0, stream, cells, planes, prop_cost, cur_cost, cur_label, W, init, flags, epoch_base,
                   rank, publish_epoch);
    return cudaGetLastError();
}

}  // namespace lexp
