// lexp_ransac.cuh -- RansacProposer on the device: RansacProposer::startIterations + getNextProposal -> RANSACPlane(coord, disps, 1.0)
// (Proposer.h:155-312) for every cell of a plan, one CTA per cell.  The contract (DESIGN.md section 3f, restated by
// tests/ransac_oracle.py):
//   * sampler: sample s of a (cell, step) takes three draws from CvRng{pm_rng_state(seed, cell_id)}, i0 = uniform_int(0, n),
//     i1 = uniform_int(0, n - 1), i2 = uniform_int(0, n - 2), mapped to three distinct row-major indices of the unit region,
//   * cv::solve(DECOMP_SVD) = the minimum-norm least-squares solution in double on the uncentred (x, y, 1) rows with the exact rank
//     of the rows (OpenCV's rule, 2 DBL_EPSILON * sum of the singular values, on integer coordinates), rounded once to float: the Gram
//     matrix of the integer coordinates exactly in int64, A^T b as a double-double sum, then a fixed sequence of IEEE double
//     operations (ransac_solve; every product and sum rounded separately; full-rank systems in coordinates centred on the unit),
//   * distances: (float)(((double)x a + (double)y b) + c) - disp in float, inlier iff |.| < 1.0f (OpenCV's float gemm accumulates
//     in double),
//   * the reference's control flow, including the refit over the inliers among the FIRST no_i points (Proposer.h:207) and
//     computeSampleCount with x86-64's double -> int conversion.
// A sample's inlier count does not depend on the running state, so the CTA counts a batch of kRansacBatch samples in one pass over
// the points, then replays the sequential acceptance in sample order (a block-wide refit only where max_i < no_i) and stops issuing
// batches once max_sam samples have been drawn: exactly the sequential result.
#pragma once

namespace lexp {

constexpr int kRansacThreads = 256;
constexpr int kRansacMaxSam = 500;                            // RansacProposer(K, MAX_SAM = 500, conf = 0.95f)
constexpr int kRansacBatch = 16;
constexpr double kRansacLog1mConf = -0x1.7f7425b73e3d1p+1;    // log(1.0 - (double)0.95f) as glibc evaluates it on the host
constexpr int kRansacJacobiSweeps = 8;

struct RansacDD { double hi, lo; };   // double-double accumulator of A^T b
__device__ __forceinline__ RansacDD dd_add(RansacDD a, double b) {   // TwoSum(a.hi, b), error into lo
    const double s = __dadd_rn(a.hi, b), bb = __dsub_rn(s, a.hi);
    const double e = __dadd_rn(__dsub_rn(a.hi, __dsub_rn(s, bb)), __dsub_rn(b, bb));
    return RansacDD{s, __dadd_rn(a.lo, e)};
}
__device__ __forceinline__ RansacDD dd_merge(RansacDD a, RansacDD b) {
    RansacDD r = dd_add(RansacDD{a.hi, 0.0}, b.hi);
    r.lo = __dadd_rn(r.lo, __dadd_rn(a.lo, b.lo));
    return r;
}

// A^T A (exact) and A^T b of the rows (x, y, 1) of a point set; h0 / h1: A^T b of the rows (x - cx, y - cy, 1), (cx, cy) = the
// integer centre of the unit region
struct RansacSys { long long xx, xy, yy, x, y, n; RansacDD g0, g1, g2, h0, h1; };
__device__ __forceinline__ void ransac_sys_add(RansacSys& s, int x, int y, float d, int cx, int cy) {
    s.xx += (long long)x * x; s.xy += (long long)x * y; s.yy += (long long)y * y; s.x += x; s.y += y; s.n++;
    const double b = (double)d;
    s.g0 = dd_add(s.g0, __dmul_rn((double)x, b));   // exact products (13-bit integer x 24-bit float)
    s.g1 = dd_add(s.g1, __dmul_rn((double)y, b));
    s.g2 = dd_add(s.g2, b);
    s.h0 = dd_add(s.h0, __dmul_rn((double)(x - cx), b));
    s.h1 = dd_add(s.h1, __dmul_rn((double)(y - cy), b));
}

// Exact rank of the rows (x, y, 1): 0 without points, 1 if all points coincide, 2 if they are collinear, else 3 (the determinant of
// the centred scatter matrix scaled by n^2, in 128-bit integers).  = ransac_oracle.gram_rank
__device__ __forceinline__ int ransac_rank(const RansacSys& s) {
    if (s.n == 0) return 0;
    const __int128 sxx = (__int128)s.n * s.xx - (__int128)s.x * s.x, syy = (__int128)s.n * s.yy - (__int128)s.y * s.y;
    const __int128 sxy = (__int128)s.n * s.xy - (__int128)s.x * s.y;
    if (sxx == 0 && syy == 0) return 1;
    return sxx * syy == sxy * sxy ? 2 : 3;
}

// The minimum-norm solution of the normal equations G N = g: cyclic Jacobi on G, then N = sum over the kept eigenpairs of
// v_i (v_i . g) / lambda_i, the 3 - rank smallest eigenvalues dropped.  Operation for operation = ransac_oracle.minnorm_solve.
__device__ LEXP_NOINLINE void ransac_minnorm(const long long G[6], const double g[3], int rank, double N[3]) {   // G: xx, xy, yy, x, y, n
    double a[3][3] = {{(double)G[0], (double)G[1], (double)G[3]}, {(double)G[1], (double)G[2], (double)G[4]}, {(double)G[3], (double)G[4], (double)G[5]}};
    double V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
    for (int sweep = 0; sweep < kRansacJacobiSweeps; sweep++)
        for (int pq = 0; pq < 3; pq++) {
            const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2, r = 3 - p - q;
            const double apq = a[p][q];
            if (apq == 0.0) continue;
            const double tau = __ddiv_rn(__dsub_rn(a[q][q], a[p][p]), __dmul_rn(2.0, apq));
            double t = __ddiv_rn(1.0, __dadd_rn(fabs(tau), sqrt(__dadd_rn(1.0, __dmul_rn(tau, tau)))));
            if (tau < 0.0) t = -t;
            const double c = __ddiv_rn(1.0, sqrt(__dadd_rn(1.0, __dmul_rn(t, t)))), sn = __dmul_rn(t, c);
            a[p][p] = __dsub_rn(a[p][p], __dmul_rn(t, apq));
            a[q][q] = __dadd_rn(a[q][q], __dmul_rn(t, apq));
            a[p][q] = a[q][p] = 0.0;
            const double arp = a[r][p], arq = a[r][q];
            a[r][p] = a[p][r] = __dsub_rn(__dmul_rn(c, arp), __dmul_rn(sn, arq));
            a[r][q] = a[q][r] = __dadd_rn(__dmul_rn(sn, arp), __dmul_rn(c, arq));
            for (int k = 0; k < 3; k++) {
                const double vkp = V[k][p], vkq = V[k][q];
                V[k][p] = __dsub_rn(__dmul_rn(c, vkp), __dmul_rn(sn, vkq));
                V[k][q] = __dadd_rn(__dmul_rn(sn, vkp), __dmul_rn(c, vkq));
            }
        }
    bool keep[3] = {true, true, true};
    for (int d = rank; d < 3; d++) {   // drop the smallest eigenvalues (the first of equal ones)
        int m = -1;
        for (int j = 0; j < 3; j++)
            if (keep[j] && (m < 0 || a[j][j] < a[m][m])) m = j;
        keep[m] = false;
    }
    N[0] = N[1] = N[2] = 0.0;
    for (int i = 0; i < 3; i++)
        if (keep[i]) {
            const double d = __dadd_rn(__dadd_rn(__dmul_rn(V[0][i], g[0]), __dmul_rn(V[1][i], g[1])), __dmul_rn(V[2][i], g[2]));
            const double w = __ddiv_rn(d, a[i][i]);
            for (int k = 0; k < 3; k++) N[k] = __dadd_rn(N[k], __dmul_rn(V[k][i], w));
        }
}

// The contract's cv::solve(DECOMP_SVD), rounded to float.  Full rank: the least-squares solution does not depend on the origin, so it
// is solved in coordinates centred on (cx, cy) (the Gram matrix of absolute coordinates squares their poor conditioning), then
// c = c' - (a cx + b cy).  Rank < 3: the minimum-norm solution of the uncentred rows, which depends on the origin.  = ransac_oracle.fit
__device__ LEXP_NOINLINE float4 ransac_solve(const RansacSys s, int cx, int cy) {
    const int rank = ransac_rank(s);
    double N[3];
    if (rank == 3) {
        const long long G[6] = {s.xx - 2 * cx * s.x + (long long)cx * cx * s.n, s.xy - cx * s.y - cy * s.x + (long long)cx * cy * s.n,
                                s.yy - 2 * cy * s.y + (long long)cy * cy * s.n, s.x - cx * s.n, s.y - cy * s.n, s.n};
        const double g[3] = {__dadd_rn(s.h0.hi, s.h0.lo), __dadd_rn(s.h1.hi, s.h1.lo), __dadd_rn(s.g2.hi, s.g2.lo)};
        ransac_minnorm(G, g, 3, N);
        N[2] = __dsub_rn(N[2], __dadd_rn(__dmul_rn(N[0], (double)cx), __dmul_rn(N[1], (double)cy)));
    } else {
        const long long G[6] = {s.xx, s.xy, s.yy, s.x, s.y, s.n};
        const double g[3] = {__dadd_rn(s.g0.hi, s.g0.lo), __dadd_rn(s.g1.hi, s.g1.lo), __dadd_rn(s.g2.hi, s.g2.lo)};
        ransac_minnorm(G, g, rank, N);
    }
    return make_float4((float)N[0], (float)N[1], (float)N[2], 0.0f);
}

// RansacProposer::computeSampleCount (Proposer.h:230-250) with conf = (double)0.95f; (int) of a quotient outside the int range or
// NaN is INT_MIN as on x86-64 (then clamped to 1)
__device__ __forceinline__ int ransac_sample_count(int ni, int pt_num) {
    double q = 1.0;
    for (double a = (double)(ni - 2), b = (double)(pt_num - 2); a <= (double)ni; a = __dadd_rn(a, 1.0), b = __dadd_rn(b, 1.0))
        q = __dmul_rn(q, __ddiv_rn(a, b));
    int cnt = 1;
    const double omq = __dsub_rn(1.0, q);
    if (!(omq < 1e-4)) {
        const double r = __ddiv_rn(kRansacLog1mConf, log(omq));
        cnt = (r > -2147483649.0 && r < 2147483648.0) ? (int)r : (-2147483647 - 1);   // INT_MIN
    }
    return cnt < 1 ? 1 : cnt;
}

__device__ __forceinline__ bool ransac_inlier(double a, double b, double c, int x, int y, float d) {
    const float pred = (float)__dadd_rn(__dadd_rn(__dmul_rn((double)x, a), __dmul_rn((double)y, b)), c);
    return fabsf(__fsub_rn(pred, d)) < 1.0f;
}

// disp_img: float[H][W] scratch; each CTA writes its unit region's snapshot there (unit regions of a plan's cells are disjoint).
// planes[call] = the proposal of the cell.  One CTA per call, kRansacThreads threads.
__global__ void __launch_bounds__(kRansacThreads) lexp_ransac_kernel(const CallInfo* __restrict__ calls, const float4* __restrict__ cur_label,
                                                                     float* __restrict__ disp_img, Plane4* __restrict__ planes, int W,
                                                                     unsigned long long seed) {
    __shared__ int s_tri[kRansacBatch][3];
    __shared__ double s_N[kRansacBatch][3];
    __shared__ int s_cnt[kRansacBatch];
    __shared__ long long s_ri[6][kRansacThreads];
    __shared__ double s_rd[10][kRansacThreads];
    __shared__ double s_fit[3];
    __shared__ int s_one;
    constexpr int T = kRansacThreads;
    const int tid = threadIdx.x;
    const CallInfo ci = calls[blockIdx.x];
    const int n = ci.uw * ci.uh;
    const int cx = ci.ux + ci.uw / 2, cy = ci.uy + ci.uh / 2;
    if (n <= 3) {   // no sample can have more than 3 inliers: Plane(0, 0, 0)
        if (tid == 0) planes[blockIdx.x] = Plane4{0.0f, 0.0f, 0.0f, 0.0f};
        return;
    }
    // startIterations: disps = (v0 x + v1 y) + v2 in float (Plane::GetZ order)
    for (int i = tid; i < n; i += T) {
        const int x = ci.ux + i % ci.uw, y = ci.uy + i / ci.uw;
        const float4 l = cur_label[(size_t)y * W + x];
        disp_img[(size_t)y * W + x] = __fadd_rn(__fadd_rn(__fmul_rn(l.x, (float)x), __fmul_rn(l.y, (float)y)), l.z);
    }
    CvRng rng{pm_rng_state(seed, ci.cell_id)};   // used by thread 0 only
    // block-wide reductions (fixed tree: the result does not depend on scheduling)
    auto reduce_sys = [&](RansacSys s) -> RansacSys {
        s_ri[0][tid] = s.xx; s_ri[1][tid] = s.xy; s_ri[2][tid] = s.yy; s_ri[3][tid] = s.x; s_ri[4][tid] = s.y; s_ri[5][tid] = s.n;
        const RansacDD* dd[5] = {&s.g0, &s.g1, &s.g2, &s.h0, &s.h1};
        for (int k = 0; k < 5; k++) { s_rd[2 * k][tid] = dd[k]->hi; s_rd[2 * k + 1][tid] = dd[k]->lo; }
        __syncthreads();
        for (int st = T / 2; st > 0; st >>= 1) {
            if (tid < st) {
                for (int k = 0; k < 6; k++) s_ri[k][tid] += s_ri[k][tid + st];
                for (int k = 0; k < 5; k++) {
                    const RansacDD m = dd_merge(RansacDD{s_rd[2 * k][tid], s_rd[2 * k + 1][tid]}, RansacDD{s_rd[2 * k][tid + st], s_rd[2 * k + 1][tid + st]});
                    s_rd[2 * k][tid] = m.hi; s_rd[2 * k + 1][tid] = m.lo;
                }
            }
            __syncthreads();
        }
        return RansacSys{s_ri[0][0], s_ri[1][0], s_ri[2][0], s_ri[3][0], s_ri[4][0], s_ri[5][0],
                         RansacDD{s_rd[0][0], s_rd[1][0]}, RansacDD{s_rd[2][0], s_rd[3][0]}, RansacDD{s_rd[4][0], s_rd[5][0]},
                         RansacDD{s_rd[6][0], s_rd[7][0]}, RansacDD{s_rd[8][0], s_rd[9][0]}};
    };
    auto count_inliers = [&](double a, double b, double c) -> int {
        __syncthreads();
        if (tid == 0) s_one = 0;
        __syncthreads();
        int k = 0;
        for (int i = tid; i < n; i += T) {
            const int x = ci.ux + i % ci.uw, y = ci.uy + i / ci.uw;
            k += ransac_inlier(a, b, c, x, y, disp_img[(size_t)y * W + x]) ? 1 : 0;
        }
        if (k) atomicAdd(&s_one, k);
        __syncthreads();
        return s_one;
    };
    int max_i = 3, max_sam = kRansacMaxSam, no_sam = 0, no_i_c = 0;
    float4 result = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    __syncthreads();   // the snapshot is complete
    while (no_sam < max_sam) {
        const int nb = min(kRansacBatch, max_sam - no_sam);
        if (tid == 0)
            for (int s = 0; s < nb; s++) {   // randperm(len)[0..2]
                int i0 = rng.uniform_int(0, n), i1 = rng.uniform_int(0, n - 1), i2 = rng.uniform_int(0, n - 2);
                i1 += i1 >= i0 ? 1 : 0;
                const int lo = min(i0, i1), hi = max(i0, i1);
                i2 += i2 >= lo ? 1 : 0;
                i2 += i2 >= hi ? 1 : 0;
                s_tri[s][0] = i0; s_tri[s][1] = i1; s_tri[s][2] = i2;
            }
        if (tid < kRansacBatch) s_cnt[tid] = 0;
        __syncthreads();
        if (tid < nb) {   // cv::solve on the three sampled rows
            RansacSys sy{0, 0, 0, 0, 0, 0, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
            for (int k = 0; k < 3; k++) {
                const int i = s_tri[tid][k], x = ci.ux + i % ci.uw, y = ci.uy + i / ci.uw;
                ransac_sys_add(sy, x, y, disp_img[(size_t)y * W + x], cx, cy);
            }
            const float4 N = ransac_solve(sy, cx, cy);
            s_N[tid][0] = (double)N.x; s_N[tid][1] = (double)N.y; s_N[tid][2] = (double)N.z;
        }
        __syncthreads();
        {   // no_i of every sample of the batch, one pass over the points
            int cnt[kRansacBatch];
#pragma unroll
            for (int s = 0; s < kRansacBatch; s++) cnt[s] = 0;
            for (int i = tid; i < n; i += T) {
                const int x = ci.ux + i % ci.uw, y = ci.uy + i / ci.uw;
                const float d = disp_img[(size_t)y * W + x];
#pragma unroll
                for (int s = 0; s < kRansacBatch; s++)
                    if (s < nb) cnt[s] += ransac_inlier(s_N[s][0], s_N[s][1], s_N[s][2], x, y, d) ? 1 : 0;
            }
#pragma unroll
            for (int s = 0; s < kRansacBatch; s++)
                if (s < nb && cnt[s]) atomicAdd(&s_cnt[s], cnt[s]);
        }
        __syncthreads();
        // the sequential acceptance, in sample order (every thread holds the same state)
        for (int s = 0; s < nb && no_sam < max_sam; s++) {
            no_sam++;
            const int no_i = s_cnt[s];
            if (max_i < no_i) {   // re-estimate on the inliers among the first no_i points (Proposer.h:203-213)
                const double a = s_N[s][0], b = s_N[s][1], c = s_N[s][2];
                RansacSys sy{0, 0, 0, 0, 0, 0, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
                for (int i = tid; i < no_i; i += T) {
                    const int x = ci.ux + i % ci.uw, y = ci.uy + i / ci.uw;
                    const float d = disp_img[(size_t)y * W + x];
                    if (ransac_inlier(a, b, c, x, y, d)) ransac_sys_add(sy, x, y, d, cx, cy);
                }
                const RansacSys tot = reduce_sys(sy);
                if (tid == 0) {
                    const float4 N = ransac_solve(tot, cx, cy);
                    s_fit[0] = (double)N.x; s_fit[1] = (double)N.y; s_fit[2] = (double)N.z;
                }
                __syncthreads();
                const double fa = s_fit[0], fb = s_fit[1], fc = s_fit[2];
                const int no = count_inliers(fa, fb, fc);
                if (no > no_i_c) {
                    result = make_float4((float)fa, (float)fb, (float)fc, 0.0f);
                    no_i_c = no;
                    max_i = no_i;
                    max_sam = min(max_sam, ransac_sample_count(no, n));
                }
            }
        }
        __syncthreads();   // s_tri / s_N / s_cnt are rewritten by the next batch
    }
    if (tid == 0) planes[blockIdx.x] = Plane4{result.x, result.y, result.z, 0.0f};
}

}  // namespace lexp
