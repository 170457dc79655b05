// lexp_post.cuh -- the post-processing of a two-view run on the device: PMStereoBase::postProcess (PMStereoBase.h:146-256), the step
// that turns the raw labelings of both views (disp0raw.pfm) into the final ones (disp0.pfm, main.cpp:319,410).
//
//   step 1  doConsistencyCheck (PMStereoBase.h:111-144)        -> lexp_post_check_kernel    (one thread per pixel, both views)
//   step 2  fail > 0, cv::dilate with a 3x3 rectangle (:162-166) -> lexp_post_fill_kernel    (one CTA per row and view)
//   step 3  horizontal nearest-neighbour fill (:169-202)       ->   "                         (two block-wide scans per row)
//   -       row-major list of the failed pixels                 -> lexp_post_offsets_kernel + lexp_post_compact_kernel
//   step 4  weighted median over (2 windR + 1)^2 (:209-252)     -> lexp_post_median_kernel   (one CTA per failed pixel)
//
// Arithmetic as in the reference: disparities are computeDisparities = channelDot((x, y, 1, 0), L) and keys Plane::GetZ, every product
// and sum rounded separately (gc_disp / gc_getz); the weights exp(-absdiff / omega) come from a table the host fills with its own
// std::exp(float) (absdiff of two 8-bit BGR pixels is an integer 0..765), so they are bit-identical to computePatchWeight; both sums of
// the weights are sequential double sums in the reference's orders (row-major total, running sum in sorted order).  The only freedom
// the reference leaves -- the order std::sort gives to equal keys -- is fixed here: candidates are sorted by (key, row-major index),
// -0 ties with +0 as under operator<, and NaN keys sort after every number.  isValid() is always true in the reference (:80-83).
// All scans are shared-memory scans (no warp shuffles), so the CPU emulator of tests/emu/ runs the same source.
#pragma once
#include "lexp_gc.cuh"

namespace lexp {

constexpr int kPostThreads = 256;        // CTA size of every post-processing kernel but the check
constexpr int kPostWeights = 766;        // absdiff of two 8-bit BGR pixels: 0 .. 3 * 255
constexpr int kPostMedianCtasPerSm = 8;  // grid of the median kernel: a grid-stride loop over the failed pixels

// Step 1 for both views (blockIdx.z = view; sign = +1 for view 0, -1 for view 1).  fail = 0 (consistent), 255 (the other view's
// disparity at rx differs by more than `threshold`) or 128 (rx outside the image).  rx = int(x - ds * sign + 0.5f) as the x86-64
// conversion cvttss2si computes it: truncation toward zero, and INT_MIN ("outside") for NaN and |v| >= 2^31 -- cvt.rzi would give 0
// for NaN and saturate large values, so those cases are taken first.  A NaN difference never fails, as in the reference.
__global__ void lexp_post_check_kernel(const float4* __restrict__ lab0, const float4* __restrict__ lab1, unsigned char* __restrict__ fail,
                                       int H, int W, float threshold) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, i = blockIdx.z;
    if (x >= W) return;
    const float4* me = i ? lab1 : lab0;
    const float4* other = i ? lab0 : lab1;
    const size_t p = (size_t)y * W + x;
    const float ds = gc_disp(me[p], (float)x, (float)y);
    const float v = __fadd_rn(__fsub_rn((float)x, __fmul_rn(ds, i ? -1.0f : 1.0f)), 0.5f);
    unsigned char f = 128;
    if (v > -2147483648.0f && v < 2147483648.0f) {
        const int rx = __float2int_rz(v);
        if (rx >= 0 && rx < W) {
            const float dsr = gc_disp(other[(size_t)y * W + rx], (float)rx, (float)y);
            f = fabsf(__fsub_rn(dsr, ds)) > threshold ? 255 : 0;
        }
    }
    fail[(size_t)i * H * W + p] = f;
}

// Inclusive scan of one int per thread over the CTA with an associative `op` (Hillis-Steele in shared memory s[blockDim.x]).
// *total = the scan of the whole CTA.  Every thread of the CTA must call it; s may be reused right after it returns.
template <class Op>
__device__ __forceinline__ int post_block_scan(int v, int* s, Op op, int* total) {
    const int t = threadIdx.x, n = blockDim.x;
    s[t] = v;
    __syncthreads();
    for (int o = 1; o < n; o <<= 1) {
        const int u = t >= o ? s[t - o] : 0;
        __syncthreads();
        if (t >= o) v = op(u, v);
        s[t] = v;
        __syncthreads();
    }
    *total = s[n - 1];
    __syncthreads();
    return v;
}
struct PostMax { __device__ __forceinline__ int operator()(int a, int b) const { return a > b ? a : b; } };
struct PostMin { __device__ __forceinline__ int operator()(int a, int b) const { return a < b ? a : b; } };
struct PostAdd { __device__ __forceinline__ int operator()(int a, int b) const { return a + b; } };

// fail2 == 0 at (x, y): no pixel of the 3x3 neighbourhood inside the image failed (cv::dilate of fail > 0 with cv::Mat() as the kernel:
// a 3x3 rectangle; the border value morphologyDefaultBorderValue never wins a maximum)
__device__ __forceinline__ bool post_fail2_zero(const unsigned char* f, int x, int y, int H, int W) {
    for (int dy = -1; dy <= 1; dy++) {
        const int yy = y + dy;
        if (yy < 0 || yy >= H) continue;
        for (int dx = -1; dx <= 1; dx++) {
            const int xx = x + dx;
            if (xx >= 0 && xx < W && f[(size_t)yy * W + xx] != 0) return false;
        }
    }
    return true;
}

// Steps 2 and 3 for row blockIdx.x of view blockIdx.y.  For every failed pixel: pl = the nearest column <= x with fail2 == 0 (a max-scan
// left to right), pr = the nearest column >= x with fail2 == 0 (a min-scan right to left); neither: unchanged, one: that one, both: pl
// if pl.GetZ(p) < pr.GetZ(p), else pr (ties and NaN take pr).  The fill reads only fail2 == 0 pixels, which it never writes.  Writes the
// filled labeling (LRcopy of the median) to `filled` and the row's number of failed pixels to counts[view * H + y].
// Dynamic shared memory: int[W] (the left scan).
__global__ void __launch_bounds__(kPostThreads) lexp_post_fill_kernel(const float4* __restrict__ lab0, const float4* __restrict__ lab1,
                                                                      const unsigned char* __restrict__ fail, float4* __restrict__ filled,
                                                                      int* __restrict__ counts, int H, int W) {
    LEXP_DYNAMIC_SMEM(smem);
    int* left = reinterpret_cast<int*>(smem);
    __shared__ int s_scan[kPostThreads];
    const int y = blockIdx.x, i = blockIdx.y, t = threadIdx.x, nt = blockDim.x;
    const size_t HW = (size_t)H * W;
    const unsigned char* f = fail + i * HW;
    const float4* lab = (i ? lab1 : lab0) + (size_t)y * W;
    const unsigned char* frow = f + (size_t)y * W;
    float4* out = filled + i * HW + (size_t)y * W;
    int carry = -1, tot = 0;
    for (int x0 = 0; x0 < W; x0 += nt) {
        const int x = x0 + t;
        int v = (x < W && post_fail2_zero(f, x, y, H, W)) ? x : -1;
        v = post_block_scan(v, s_scan, PostMax(), &tot);
        if (x < W) left[x] = v > carry ? v : carry;
        carry = tot > carry ? tot : carry;
    }
    __syncthreads();
    int carry_r = W, count = 0;
    for (int x1 = W - 1; x1 >= 0; x1 -= nt) {
        const int x = x1 - t;   // thread t scans column x1 - t: an inclusive scan over t runs right to left
        int v = (x >= 0 && post_fail2_zero(f, x, y, H, W)) ? x : W;
        v = post_block_scan(v, s_scan, PostMin(), &tot);
        const int r = v < carry_r ? v : carry_r;
        carry_r = tot < carry_r ? tot : carry_r;
        if (x >= 0) {
            float4 L = lab[x];
            if (frow[x] != 0) {
                count++;
                const int l = left[x];
                if (l >= 0 && r < W) {
                    const float4 pl = lab[l], pr = lab[r];
                    L = gc_getz(pl, (float)x, (float)y) < gc_getz(pr, (float)x, (float)y) ? pl : pr;
                } else if (l >= 0) L = lab[l];
                else if (r < W) L = lab[r];
            }
            out[x] = L;
        }
    }
    post_block_scan(count, s_scan, PostAdd(), &tot);
    if (t == 0) counts[i * H + y] = tot;
}

// offsets[k] = counts[0] + .. + counts[k - 1] for k = 0 .. n (one CTA)
__global__ void __launch_bounds__(kPostThreads) lexp_post_offsets_kernel(const int* __restrict__ counts, int n, int* __restrict__ offsets) {
    __shared__ int s_scan[kPostThreads];
    int carry = 0, tot = 0;
    for (int k0 = 0; k0 < n; k0 += blockDim.x) {
        const int k = k0 + threadIdx.x;
        const int v = k < n ? counts[k] : 0;
        const int inc = post_block_scan(v, s_scan, PostAdd(), &tot);
        if (k < n) offsets[k] = carry + inc - v;
        carry += tot;
    }
    if (threadIdx.x == 0) offsets[n] = carry;
}

// The failed pixels of row blockIdx.x of view blockIdx.y, in row-major order, at list[offsets[view * H + y] ..] as view * H * W + y * W + x
__global__ void __launch_bounds__(kPostThreads) lexp_post_compact_kernel(const unsigned char* __restrict__ fail, const int* __restrict__ offsets,
                                                                         int* __restrict__ list, int H, int W) {
    __shared__ int s_scan[kPostThreads];
    const int y = blockIdx.x, i = blockIdx.y;
    const size_t row = (size_t)i * H * W + (size_t)y * W;
    int at = offsets[i * H + y], tot = 0;
    for (int x0 = 0; x0 < W; x0 += blockDim.x) {
        const int x = x0 + threadIdx.x;
        const int flag = x < W && fail[row + x] != 0;
        const int inc = post_block_scan(flag, s_scan, PostAdd(), &tot);
        if (flag) list[at + inc - 1] = (int)(row + x);
        at += tot;
    }
}

// Sort key of a median candidate: the order of the float key (operator<), -0 equal to +0, NaN after every number.  The low 32 bits of
// an entry hold the candidate's row-major index in the window, so equal keys keep that order.
__device__ __forceinline__ unsigned post_sort_key(float z) {
    if (z != z) return 0xFFFFFFFFu;
    const unsigned u = __float_as_uint(z == 0.0f ? 0.0f : z);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Step 4 for the failed pixels list[0 .. *n_list) (grid-stride, one pixel per CTA at a time).  The window is
// getLargerRect(p, windR) & imageDomain; candidate q (row-major index k) has key filled(q).GetZ(p) and weight wtab[absdiff(I(p), I(q))].
// The result is the first candidate, in (key, k) order, whose running double sum of weights exceeds half the row-major double total;
// it is copied from `filled` (never from the state being written) into the state of the view.  Without a crossing the pixel keeps its
// filled label, as the reference keeps its hole-filled one.  Dynamic shared memory: u64[npow2] entries, float[(2 windR + 1)^2] weights.
__global__ void __launch_bounds__(kPostThreads) lexp_post_median_kernel(const float4* __restrict__ filled, const uchar4* __restrict__ guide0,
                                                                        const uchar4* __restrict__ guide1, const float* __restrict__ wtab,
                                                                        const int* __restrict__ list, const int* __restrict__ n_list,
                                                                        float4* lab0, float4* lab1, int H, int W, int windR, int npow2) {
    LEXP_DYNAMIC_SMEM(smem);
    u64* ent = reinterpret_cast<u64*>(smem);
    float* wt = reinterpret_cast<float*>(ent + npow2);
    const int t = threadIdx.x, nt = blockDim.x;
    const int total = *n_list;
    const size_t HW = (size_t)H * W;
    for (int j = blockIdx.x; j < total; j += gridDim.x) {
        const int e = list[j];
        const int i = (size_t)e >= HW ? 1 : 0;
        const int p = (int)(e - i * HW);
        const int x = p % W, y = p / W;
        const int x0 = max(x - windR, 0), x1 = min(x + windR + 1, W), y0 = max(y - windR, 0), y1 = min(y + windR + 1, H);
        const int w = x1 - x0, n = w * (y1 - y0);
        const float4* src = filled + i * HW;
        const uchar4* g = i ? guide1 : guide0;
        const uchar4 gp = g[p];
        for (int k = t; k < npow2; k += nt) {
            if (k < n) {
                const size_t q = (size_t)(y0 + k / w) * W + (x0 + k % w);
                const uchar4 gq = g[q];
                const int ad = abs((int)gp.x - (int)gq.x) + abs((int)gp.y - (int)gq.y) + abs((int)gp.z - (int)gq.z);
                wt[k] = wtab[ad];
                ent[k] = ((u64)post_sort_key(gc_getz(src[q], (float)x, (float)y)) << 32) | (unsigned)k;
            } else ent[k] = ~0ull;   // padding to a power of two: after every candidate
        }
        __syncthreads();
        for (int size = 2; size <= npow2; size <<= 1)   // bitonic sort, ascending
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int k = t; k < npow2 / 2; k += nt) {
                    const int lo = 2 * k - (k & (stride - 1)), hi = lo + stride;
                    const bool up = (lo & size) == 0;
                    const u64 a = ent[lo], b = ent[hi];
                    if ((a > b) == up) { ent[lo] = b; ent[hi] = a; }
                }
                __syncthreads();
            }
        if (t == 0) {
            double sumw = 0.0;   // sumw of :220, in row-major order
            for (int k = 0; k < n; k++) sumw = __dadd_rn(sumw, (double)wt[k]);
            const double center = sumw / 2.0;
            double run = 0.0;
            int pick = -1;
            for (int k = 0; k < n; k++) {
                const int c = (int)(unsigned)ent[k];
                run = __dadd_rn(run, (double)wt[c]);
                if (run > center) { pick = c; break; }
            }
            float4* dst = i ? lab1 : lab0;
            dst[p] = pick >= 0 ? src[(size_t)(y0 + pick / w) * W + (x0 + pick % w)] : src[p];
        }
        __syncthreads();   // ent / wt are rewritten for the next pixel
    }
}

}  // namespace lexp
