// lexp_label_cost.cuh -- initCurrentFast started from a given labeling (FastGCStereo.h:116-130) on the device: for every pixel p of
// one view
//   currentCost_(p) = ComputeUnaryPotential(F(p), {p}, ., currentLabeling_(p)),   F(p) = (p.x - windR, p.y - windR, 2 windR + 1,
//   2 windR + 1) & image,
// the check version with the 1x1 fast path of IsValiLabel (StereoEnergy.h:560-583).  The contract is DESIGN.md section 3g.
//
// windR >= 2R (R = windR / 2), so for every k of the box w(p) the box w(k) lies inside p +- 2R, hence inside F(p) once clipped to the
// image: every window count is the image-clipped count, and only the (4R+1)^2 raw samples around p enter the result.  The raw cost
// is still that of F(p): for the cost-volume energy it does not depend on F, but NaiveStereoEnergy builds its warp's affine map from
// F(p)'s corners with fixed-point coordinates relative to F(p)'s origin (StereoEnergy.h:704-729), so that map is built per pixel.
//
// Every pixel has its own plane, so nothing is shared between pixels: one CTA of kLcThreads per output pixel.
//   1. raw samples of the (4R+1)^2 window around p -> shared memory (0 outside the image: the box filter's zero padding);
//   2. a thread per window column: its sums of {p, I0 p, I1 p, I2 p} over 2R+1 rows, centred on each of the 2R+1 rows of w(p);
//   3. every point k of w(p) inside the image: box sums = 2R+1 column sums, (a, b) from the statistics (GuidedFilter.h:206-220);
//      each thread sums the (a, b) of its points in a fixed order;
//   4. a fixed-shape tree reduction in shared memory, q = (sum b + sum a . I(p)) / N(p) (GuidedFilter.h:224-243), validity mask.
// Raw costs use team A's arithmetic of lexp_fused_kernel (every product and sum rounded separately); the filter runs in FP32.  No
// atomics and no warp-level exchange: two calls give the same bits.
#pragma once

namespace lexp {

constexpr int kLcThreads = 128;

struct LcParams {
    const float* __restrict__ vol;        // blocked cost volume of the view (as KParams::vol)
    int Wb;
    const uchar4* __restrict__ guide;
    const float4* __restrict__ statA;
    const float4* __restrict__ statB;
    const float* __restrict__ statC;
    const float4* __restrict__ exi_own;   // NaiveStereoEnergy: ExI[mode], ExI[1 - mode]
    const float4* __restrict__ exi_other;
    const float4* __restrict__ label;     // currentLabeling_[mode], read only
    float* __restrict__ cost;             // currentCost_[mode]
    int H, W, D, R, windR, mode;
    float th_col, min_disp, max_disp, thresh_color, thresh_gradient;
};

// dynamic shared memory: column sums float4[2R+1][4R+1], reduction float4[kLcThreads], the inverse affine map double[6], raw samples
// float[4R+1][4R+1], the fixed-point row / column terms of the naive warp int[4][4R+1]
__host__ __device__ inline size_t label_cost_smem_bytes(int R) {
    const size_t NW = 4 * R + 1, K = 2 * R + 1;
    return K * NW * 16 + (size_t)kLcThreads * 16 + 6 * 8 + NW * NW * 4 + 4 * NW * 4;
}

// CostVolumeEnergy raw cost of plane pl at (x, y) (CostVolumeEnergy.h:69-98): the generic sampler of lexp_fused_kernel's team A
__device__ __forceinline__ float lc_raw_volume(const LcParams& P, const Plane4 pl, int x, int y) {
    const float d = __fadd_rn(__fmul_rn(pl.a, (float)x), __fadd_rn(__fmul_rn(pl.b, (float)y), pl.c));   // :73, :76
    const bool lo = d < P.min_disp;                                    // :78
    const bool hi = !lo && d >= P.max_disp;                            // :79
    bool bad = !lo && !hi && (isnan(d) || isinf(d));                   // :80
    const float dd = (lo || hi || bad) ? 0.f : d;
    const int d0 = (int)dd + (int)(-P.min_disp);                       // :83
    const float f1 = dd - floorf(dd);                                  // :85
    if (d0 + 1 >= P.D || d0 < 0) bad = true;                           // :87-90
    // blocked volume: element (d, y, x) at ((((y/4) * Wb + x/4) * D + d) * 4 + y%4) * 4 + x%4
    const float* blk = P.vol + ((size_t)(y >> 2) * P.Wb + (x >> 2)) * P.D * 16 + (y & 3) * 4 + (x & 3);
    float C;
    if (lo) C = __ldg(blk);
    else if (hi) C = __ldg(blk + (size_t)(P.D - 1) * 16);
    else if (bad) C = kCostInvalid;
    else C = __fadd_rn(__fmul_rn(1.0f - f1, __ldg(blk + (size_t)d0 * 16)), __fmul_rn(f1, __ldg(blk + (size_t)(d0 + 1) * 16)));   // :92
    return (P.th_col < C) ? P.th_col : C;                              // std::min (:96)
}

// NaiveStereoEnergy raw cost at (x, y) (StereoEnergy.h:729-741): X, Y = cv::warpAffine's fixed-point source coordinates (before the
// final >> 5), as team A's NAIVE path of lexp_fused_kernel computes them
__device__ __forceinline__ float lc_raw_naive(const LcParams& P, int x, int y, int Xf, int Yf) {
    const int X = Xf >> 5, Y = Yf >> 5;
    const int sx = X >> 5, sy = Y >> 5;
    const float fxw = (float)(X & 31) * (1.0f / 32), fyw = (float)(Y & 31) * (1.0f / 32);
    const int Wm1 = P.W - 1, Hm1 = P.H - 1;
    const int x0c = min(max(sx, 0), Wm1), x1c = min(max(sx + 1, 0), Wm1);
    const int y0c = min(max(sy, 0), Hm1), y1c = min(max(sy + 1, 0), Hm1);
    const float4 S00 = __ldg(P.exi_other + (size_t)y0c * P.W + x0c), S01 = __ldg(P.exi_other + (size_t)y0c * P.W + x1c);
    const float4 S10 = __ldg(P.exi_other + (size_t)y1c * P.W + x0c), S11 = __ldg(P.exi_other + (size_t)y1c * P.W + x1c);
    const float4 L = __ldg(P.exi_own + (size_t)y * P.W + x);
    const float w00 = __fmul_rn(1.0f - fyw, 1.0f - fxw), w01 = __fmul_rn(1.0f - fyw, fxw);
    const float w10 = __fmul_rn(fyw, 1.0f - fxw), w11 = __fmul_rn(fyw, fxw);
    auto bil = [&](float a, float b, float cc, float d) {  // remapBilinear: ((S00 w00 + S01 w01) + S10 w10) + S11 w11
        return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, w00), __fmul_rn(b, w01)), __fmul_rn(cc, w10)), __fmul_rn(d, w11));
    };
    const float r0 = bil(S00.x, S01.x, S10.x, S11.x), r1 = bil(S00.y, S01.y, S10.y, S11.y);
    const float r2 = bil(S00.z, S01.z, S10.z, S11.z), r3 = bil(S00.w, S01.w, S10.w, S11.w);
    const float col = __fadd_rn(__fadd_rn(fabsf(__fsub_rn(L.x, r0)), fabsf(__fsub_rn(L.y, r1))), fabsf(__fsub_rn(L.z, r2)));
    return __fadd_rn(fminf(P.thresh_color, col), fminf(P.thresh_gradient, fabsf(__fsub_rn(L.w, r3))));   // :737-740
}

__device__ __forceinline__ float4 lc_add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

// grid = (W, H): block (x, y) computes currentCost_(x, y)
template <bool NAIVE>
__global__ void __launch_bounds__(kLcThreads) lexp_label_cost_kernel(const LcParams P) {
    const int R = P.R, K = 2 * R + 1, NW = 4 * R + 1;
    const int H = P.H, W = P.W;
    const int px = blockIdx.x, py = blockIdx.y, tid = threadIdx.x;
    const int X0 = px - 2 * R, Y0 = py - 2 * R;   // image coordinates of window column / row 0
    LEXP_DYNAMIC_SMEM(smem_raw);
    float4* s_col = reinterpret_cast<float4*>(smem_raw);             // [K][NW]: column sums centred on row py - R + jc
    float4* s_red = s_col + K * NW;                                   // [kLcThreads]
    double* s_iM = reinterpret_cast<double*>(s_red + kLcThreads);     // [6]
    float* s_p = reinterpret_cast<float*>(s_iM + 6);                  // [NW][NW] raw samples
    int* s_rx = reinterpret_cast<int*>(s_p + NW * NW);                // NAIVE [NW] x 4: fixed-point row terms / column deltas
    int* s_ry = s_rx + NW;
    int* s_ca = s_ry + NW;
    int* s_cb = s_ca + NW;
    const size_t pix = (size_t)py * W + px;
    const float4 l4 = P.label[pix];
    const Plane4 pl{l4.x, l4.y, l4.z, l4.w};

    if (NAIVE) {
        // the warp of F(p): the reference's filterRegion of a 1x1 unit (FastGCStereo.h:120-129)
        Item it{};
        it.fx = max(px - P.windR, 0); it.fy = max(py - P.windR, 0);
        it.fw = min(px + P.windR + 1, W) - it.fx; it.fh = min(py + P.windR + 1, H) - it.fy;
        if (tid == 0) naive_inverse_affine(it, pl, P.mode, s_iM);
        __syncthreads();
        // cv::warpAffine fixed-point terms (AB_BITS = 10, round_delta = 16), relative to F(p)'s origin
        for (int j = tid; j < NW; j += kLcThreads) {
            const double yr = (double)(Y0 + j - it.fy), xr = (double)(X0 + j - it.fx);
            s_rx[j] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(s_iM[1], yr), s_iM[2]), 1024.0)) + 16;
            s_ry[j] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(s_iM[4], yr), s_iM[5]), 1024.0)) + 16;
            s_ca[j] = __double2int_rn(__dmul_rn(__dmul_rn(s_iM[0], xr), 1024.0));
            s_cb[j] = __double2int_rn(__dmul_rn(__dmul_rn(s_iM[3], xr), 1024.0));
        }
        __syncthreads();
    }

    // 1. raw samples of the window (inside the image they all lie inside F(p))
    for (int i = tid; i < NW * NW; i += kLcThreads) {
        const int j = i / NW, ii = i - j * NW;
        const int y = Y0 + j, x = X0 + ii;
        float p = 0.f;
        if (y >= 0 && y < H && x >= 0 && x < W) {
            if (NAIVE) p = lc_raw_naive(P, x, y, s_rx[j] + s_ca[ii], s_ry[j] + s_cb[ii]);
            else p = lc_raw_volume(P, pl, x, y);
        }
        s_p[i] = p;
    }
    __syncthreads();

    // 2. column sums of {p, I0 p, I1 p, I2 p} (I = guide / 255) over 2R+1 rows: a running sum down the window column
    const float s255 = 1.0f / 255.0f;
    for (int ii = tid; ii < NW; ii += kLcThreads) {
        const int x = X0 + ii;
        const bool colin = x >= 0 && x < W;
        auto prod = [&](int j) {
            const float p = s_p[j * NW + ii];
            const int y = Y0 + j;
            if (!colin || y < 0 || y >= H) return make_float4(0.f, 0.f, 0.f, 0.f);
            const uchar4 g = __ldg(P.guide + (size_t)y * W + x);
            const float ps = __fmul_rn(p, s255);
            return make_float4(p, __fmul_rn((float)g.x, ps), __fmul_rn((float)g.y, ps), __fmul_rn((float)g.z, ps));
        };
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j = 0; j < NW; j++) {
            const float4 nw = prod(j);
            if (j >= K) {
                const float4 old = prod(j - K);
                acc = lc_add(acc, make_float4(nw.x - old.x, nw.y - old.y, nw.z - old.z, nw.w - old.w));
            } else acc = lc_add(acc, nw);
            if (j >= 2 * R) s_col[(j - 2 * R) * NW + ii] = acc;
        }
    }
    __syncthreads();

    // 3. (a, b) at every point k of w(p) inside the image (GuidedFilter.h:206-220), summed per thread in a fixed order
    float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = tid; k < K * K; k += kLcThreads) {
        const int jc = k / K, ic = k - jc * K;
        const int ky = py - R + jc, kx = px - R + ic;
        if (ky < 0 || ky >= H || kx < 0 || kx >= W) continue;
        const float4* cs = s_col + jc * NW + ic;
        float4 B = cs[0];
        for (int m = 1; m < K; m++) B = lc_add(B, cs[m]);
        const float invN = (1.0f / (float)(min(kx + R, W - 1) - max(kx - R, 0) + 1)) *
                           (1.0f / (float)(min(ky + R, H - 1) - max(ky - R, 0) + 1));   // GuidedFilter.h:324, image-clipped
        const size_t kp = (size_t)ky * W + kx;
        const float4 sa = __ldg(P.statA + kp), sb = __ldg(P.statB + kp);
        const float m0 = sa.x, m1 = sa.y, m2 = sa.z, i00 = sa.w;
        const float i01 = sb.x, i02 = sb.y, i11 = sb.z, i12 = sb.w, i22 = __ldg(P.statC + kp);
        const float mp = B.x * invN;                      // :206
        const float c0 = fmaf(B.y, invN, -m0 * mp);       // :212-214
        const float c1 = fmaf(B.z, invN, -m1 * mp);
        const float c2 = fmaf(B.w, invN, -m2 * mp);
        const float a0 = i00 * c0 + i01 * c1 + i02 * c2;  // :216-218
        const float a1 = i01 * c0 + i11 * c1 + i12 * c2;
        const float a2 = i02 * c0 + i12 * c1 + i22 * c2;
        const float bb = mp - a0 * m0 - a1 * m1 - a2 * m2;  // :220
        sum = lc_add(sum, make_float4(a0, a1, a2, bb));
    }
    s_red[tid] = sum;
    __syncthreads();

    // 4. fixed-shape tree reduction, output and validity
    for (int s = kLcThreads / 2; s > 0; s >>= 1) {
        if (tid < s) s_red[tid] = lc_add(s_red[tid], s_red[tid + s]);
        __syncthreads();
    }
    if (tid == 0) {
        const float4 S = s_red[0];
        const uchar4 g = __ldg(P.guide + pix);
        const float dot = S.x * (float)g.x + S.y * (float)g.y + S.z * (float)g.z;
        const float invN = (1.0f / (float)(min(px + R, W - 1) - max(px - R, 0) + 1)) * (1.0f / (float)(min(py + R, H - 1) - max(py - R, 0) + 1));
        float q = fmaf(dot, s255, S.w) * invN;   // GuidedFilter.h:243
        // IsValiLabel(Plane, Point) (StereoEnergy.h:560-583): the plane at p and at p +- (5, 5) inside [MIN, MAX]
        const float ds = __fadd_rn(__fadd_rn(__fmul_rn((float)px, pl.a), __fmul_rn((float)py, pl.b)), pl.c);
        const float a5 = __fmul_rn(pl.a, 5.0f), b5 = __fmul_rn(pl.b, 5.0f);
        const float lo = P.min_disp, hi = P.max_disp;
        const float dpp = __fadd_rn(__fadd_rn(ds, a5), b5), dpm = __fsub_rn(__fadd_rn(ds, a5), b5);
        const float dmp = __fadd_rn(__fsub_rn(ds, a5), b5), dmm = __fsub_rn(__fsub_rn(ds, a5), b5);
        const bool ok = ds >= lo && ds <= hi && dpp >= lo && dpp <= hi && dpm >= lo && dpm <= hi && dmp >= lo && dmp <= hi &&
                        dmm >= lo && dmm <= hi;
        if (!ok) q = kCostInvalid;   // CostVolumeEnergy.h:180-182
        P.cost[pix] = q;
    }
}

}  // namespace lexp
