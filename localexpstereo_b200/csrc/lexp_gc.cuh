// lexp_gc.cuh -- pairwise terms and the expansion move (graph cut) of the local expansion loop on the device.
//
// SURVEY.md section 8(f):
//   f-2  StereoEnergy::initSmoothnessCoeff            (StereoEnergy.h:131-163)  -> lexp_smooth_coeff_kernel
//        StereoEnergy::computeSmoothnessTermsExpansion (StereoEnergy.h:398-453)  -> pair_terms() / lexp_pairwise_kernel
//        StereoEnergy::computeSmoothnessTerm           (StereoEnergy.h:234-239)  -> boundary_term()
//        StereoEnergy::computeSmoothnessCost           (StereoEnergy.h:165-199)  -> lexp_energy_kernel
//   f-3  FastGCStereo::expansionMoveBK                 (FastGCStereo.h:411-597)  -> gc_node_* steps, run by lexp_gc_move_kernel (one CTA per
//                                                                                   cell) or lexp_gc_phase_kernel (large cells, all SMs)
//        FastGCStereo::initCurrentFast                 (FastGCStereo.h:101-113)  -> lexp_gc_assign_kernel (any energy kind)
//        (graph construction as there; the minimum cut itself is computed by a deterministic push-relabel instead of the un-vendored
//         Boykov-Kolmogorov library -- the segmentation BK reports, `what_segment() == SOURCE`, is the complement of the set of nodes
//         from which the sink is reachable in the residual graph of a maximum flow, which is the same set for every maximum flow)
// File:line citations are relative to /root/reference/LocalExpansionStereo/.
//
// Neighbour directions (the reference's StereoEnergy::NB_* order is LE GE EL EG LL GL LG GG, StereoEnergy.h:47-56): here
//   d = 0 GE (+1, 0)   1 EG (0,+1)   2 LG (-1,+1)   3 GG (+1,+1)        the four FORWARD neighbours (the only ones that carry edges)
//   d = 4 LE (-1, 0)   5 EL (0,-1)   6 GL (+1,-1)   7 LL (-1,-1)        their opposites: opp(d) = d ^ 4
// The coefficient of a backward neighbour equals the forward coefficient stored at that neighbour (|I(p) - I(q)| is symmetric and the
// same pixels are zeroed at the image border), so one float4 per pixel {GE, EG, LG, GG} holds all eight maps of smoothnessCoeff[mode].
#pragma once
#include "lexp_kernels.cuh"

namespace lexp {

__host__ __device__ __forceinline__ int gc_dx(int d) { return d == 0 || d == 3 || d == 6 ? 1 : (d == 1 || d == 5 ? 0 : -1); }
__host__ __device__ __forceinline__ int gc_dy(int d) { return d == 0 || d == 4 ? 0 : (d >= 1 && d <= 3 ? 1 : -1); }
// index of direction d in the reference's neighbour list (StereoEnergy.h:47-56)
__host__ __device__ __forceinline__ int gc_ref_index(int d) {
    return d == 0 ? 1 : d == 1 ? 3 : d == 2 ? 6 : d == 3 ? 7 : d == 4 ? 0 : d == 5 ? 2 : d == 6 ? 5 : 4;
}
constexpr int kGcInf = 1 << 30;     // height of a node from which the sink cannot be reached
constexpr int kGcWords = 28;        // scratch words per node: excess, sink capacity, height, 8 residual capacities, 2 x 8 push slots, proposed height

// ---- f-2: smoothness coefficients --------------------------------------------------------------------------------------------
// smoothnessCoeff[mode][k](p) = max(epsilon, exp(-sum_c |I_c(p + n_k) - I_c(p)| / omega)), zero where p + n_k lies outside the image
// (StereoEnergy.h:140-156).  The guide is 8-bit, so the channel sum is an exact integer in float.
__global__ void lexp_smooth_coeff_kernel(const uchar4* __restrict__ guide, float4* __restrict__ coef, int H, int W, float omega, float epsilon) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const uchar4 g = guide[(size_t)y * W + x];
    float v[4];
#pragma unroll
    for (int d = 0; d < 4; d++) {
        const int qx = x + gc_dx(d), qy = y + gc_dy(d);
        v[d] = 0.0f;
        if (qx >= 0 && qx < W && qy < H) {
            const uchar4 q = guide[(size_t)qy * W + qx];
            const float s = (float)(abs((int)q.x - (int)g.x) + abs((int)q.y - (int)g.y) + abs((int)q.z - (int)g.z));
            v[d] = fmaxf(epsilon, expf(-s / omega));
        }
    }
    coef[(size_t)y * W + x] = make_float4(v[0], v[1], v[2], v[3]);
}
// planar float[8][H][W] view in the reference's neighbour order (lexp_get_smooth_coeff)
__global__ void lexp_smooth_coeff_unpack(const float4* __restrict__ coef, float* __restrict__ out8, int H, int W) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const size_t HW = (size_t)H * W, p = (size_t)y * W + x;
#pragma unroll
    for (int d = 0; d < 8; d++) {
        float v;
        if (d < 4) { const float4 c = coef[p]; v = d == 0 ? c.x : d == 1 ? c.y : d == 2 ? c.z : c.w; }
        else {   // backward neighbour q = p + n_d: the forward coefficient d - 4 stored at q
            const int qx = x + gc_dx(d), qy = y + gc_dy(d);
            v = 0.0f;
            if (qx >= 0 && qx < W && qy >= 0) { const float4 c = coef[(size_t)qy * W + qx]; v = d == 4 ? c.x : d == 5 ? c.y : d == 6 ? c.z : c.w; }
        }
        out8[gc_ref_index(d) * HW + p] = v;
    }
}

// disparity of label L at the image point (x, y): cvutils::channelDot(label, coord) with coord = (x, y, 1, 0) -- the 4-term row sum of
// cv::reduce, every product and sum rounded separately (Utilities.hpp:215-229; the same order as the validity test of the unary path)
__device__ __forceinline__ float gc_disp(const float4 L, float x, float y) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(L.x, x), __fmul_rn(L.y, y)), L.z), __fmul_rn(L.w, 0.0f));
}
struct PairTerms { float c00, c01, c10; };
// One neighbour pair of computeSmoothnessTermsExpansion (StereoEnergy.h:425-451): ee = p, le = q = p + n.  L0p / L0q: current labels at
// p / q, l1: the proposal.  q outside the image: the margin of labeling_m and coordinates_m is zero (PMStereoBase.h:44, StereoEnergy.h:88),
// so every disparity "at le" or "of le" is 0 -- and so is the coefficient.
__device__ __forceinline__ PairTerms pair_terms(const float4 L0p, float4 L0q, const float4 l1, int px, int py, int qx, int qy, bool q_inside,
                                                float coef, float lambda, float th) {
    const float fx = (float)px, fy = (float)py;
    float gx = (float)qx, gy = (float)qy;
    const float d0ee_ee = gc_disp(L0p, fx, fy), d1_ee = gc_disp(l1, fx, fy);
    float d0le_ee, d0ee_le, d0le_le, d1_le;
    if (q_inside) {
        d0le_ee = gc_disp(L0q, fx, fy); d0ee_le = gc_disp(L0p, gx, gy); d0le_le = gc_disp(L0q, gx, gy); d1_le = gc_disp(l1, gx, gy);
    } else { d0le_ee = 0.0f; d0ee_le = 0.0f; d0le_le = 0.0f; d1_le = 0.0f; }
    auto term = [&](float a0, float a1, float b0, float b1) {
        float c = __fadd_rn(fabsf(__fsub_rn(a0, a1)), fabsf(__fsub_rn(b0, b1)));
        c = c > th ? th : c;                                   // cv::threshold THRESH_TRUNC
        return __fmul_rn(__fmul_rn(lambda, c), coef);          // Mat::mul(coeff, lambda): (scale * a) * b
    };
    PairTerms t;
    t.c00 = term(d0ee_ee, d0le_ee, d0ee_le, d0le_le);          // :441
    t.c01 = term(d0ee_ee, d1_ee, d0ee_le, d1_le);              // :445
    t.c10 = term(d1_ee, d0le_ee, d1_le, d0le_le);              // :449
    return t;
}
// StereoEnergy::computeSmoothnessTerm(ls, lt, ps, neighborId, mode) (StereoEnergy.h:234-239), used for the region's outer boundary
// (FastGCStereo.h:455-470):  coeff * min(|ls(ps) - lt(ps)| + |ls(pt) - lt(pt)|, th_smooth) * lambda  with Plane::GetZ = a x + b y + c
__device__ __forceinline__ float gc_getz(const float4 L, float x, float y) { return __fadd_rn(__fadd_rn(__fmul_rn(L.x, x), __fmul_rn(L.y, y)), L.z); }
__device__ __forceinline__ float boundary_term(const float4 ls, const float4 lt, int px, int py, int qx, int qy, float coef, float lambda, float th) {
    const float s = __fadd_rn(fabsf(__fsub_rn(gc_getz(ls, (float)px, (float)py), gc_getz(lt, (float)px, (float)py))),
                              fabsf(__fsub_rn(gc_getz(ls, (float)qx, (float)qy), gc_getz(lt, (float)qx, (float)qy))));
    return __fmul_rn(__fmul_rn(coef, fminf(s, th)), lambda);
}
__device__ __forceinline__ float coef_of(const float4 c, int d) { return d == 0 ? c.x : d == 1 ? c.y : d == 2 ? c.z : c.w; }

// StereoEnergy::computeSmoothnessCost (StereoEnergy.h:165-199) and the data term next to it: per pixel the float sum of cost00 over the
// forward neighbours in the reference's order (GE, EG, LG, GG: the `cv::add(sumCost, cost00_nb, sumCost)` loop), then sums in double --
// block-wise here, the blocks added up in order by lexp_energy_finish (deterministic).  part[2 b] = data, part[2 b + 1] = smoothness.
__global__ void lexp_energy_kernel(const float* __restrict__ cur_cost, const float4* __restrict__ cur_label, const float4* __restrict__ coef,
                                   double* __restrict__ part, int H, int W, float lambda, float th) {
    __shared__ double s_d[256], s_s[256];
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    double dv = 0.0, sv = 0.0;
    if (p < (long long)H * W) {
        const int X = (int)(p % W), Y = (int)(p / W);
        dv = (double)cur_cost[p];
        const float4 L0p = cur_label[p];
        const float4 cf = coef[p];
        float sum = 0.0f;
#pragma unroll
        for (int d = 0; d < 4; d++) {
            const int QX = X + gc_dx(d), QY = Y + gc_dy(d);
            const bool inside = QX >= 0 && QX < W && QY < H;
            const float4 L0q = inside ? cur_label[(size_t)QY * W + QX] : make_float4(0.f, 0.f, 0.f, 0.f);
            sum = __fadd_rn(sum, pair_terms(L0p, L0q, L0p, X, Y, QX, QY, inside, coef_of(cf, d), lambda, th).c00);
        }
        sv = (double)sum;
    }
    s_d[threadIdx.x] = dv; s_s[threadIdx.x] = sv;
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (int i = 0; i < (int)blockDim.x; i++) { a += s_d[i]; b += s_s[i]; }
        part[2 * (size_t)blockIdx.x] = a; part[2 * (size_t)blockIdx.x + 1] = b;
    }
}
__global__ void lexp_energy_finish(const double* __restrict__ part, int nblocks, double* __restrict__ out2) {
    double a = 0.0, b = 0.0;
    for (int i = 0; i < nblocks; i++) { a += part[2 * (size_t)i]; b += part[2 * (size_t)i + 1]; }
    out2[0] = a; out2[1] = b;
}

// StereoEnergy::computeDisparities(labeling) = channelDot(coordinates, labeling) (StereoEnergy.h:269-272): the disparity map the
// reference writes as disp0.pfm (main.cpp:319,410)
__global__ void lexp_disparity_kernel(const float4* __restrict__ cur_label, float* __restrict__ disp, int H, int W) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const size_t p = (size_t)y * W + x;
    disp[p] = gc_disp(cur_label[p], (float)x, (float)y);
}

struct GcCell {       // one expansion move = one cell of the group (region = its sharedRegion)
    int x, y, w, h;   // region (image coordinates)
    long long node0;  // first node of the region in the scratch arrays
};

// f-2 as an operator of its own: the three maps of computeSmoothnessTermsExpansion(.., onlyForward = true) for n (region, proposal) pairs.
// out: per call a block float[3][4][h][w] (cost00, cost01, cost10 x directions GE, EG, LG, GG) at float offset 12 * node0.
__global__ void lexp_pairwise_kernel(const GcCell* __restrict__ cells, const Plane4* __restrict__ planes, const float4* cur_label,
                                     const float4* __restrict__ coef, float* __restrict__ out, int H, int W, float lambda, float th) {
    const GcCell c = cells[blockIdx.x];
    const Plane4 pl = planes[blockIdx.x];
    const float4 l1 = make_float4(pl.a, pl.b, pl.c, pl.v);
    const int N = c.w * c.h;
    float* o = out + 12 * c.node0;
    for (int s = threadIdx.x; s < N; s += blockDim.x) {
        const int x = s % c.w, y = s / c.w, X = c.x + x, Y = c.y + y;
        const float4 L0p = cur_label[(size_t)Y * W + X];
        const float4 cf = coef[(size_t)Y * W + X];
#pragma unroll
        for (int d = 0; d < 4; d++) {
            const int QX = X + gc_dx(d), QY = Y + gc_dy(d);
            const bool inside = QX >= 0 && QX < W && QY < H;
            const float4 L0q = inside ? cur_label[(size_t)QY * W + QX] : make_float4(0.f, 0.f, 0.f, 0.f);
            const PairTerms t = pair_terms(L0p, L0q, l1, X, Y, QX, QY, inside, coef_of(cf, d), lambda, th);
            o[(size_t)(0 * 4 + d) * N + s] = t.c00;
            o[(size_t)(1 * 4 + d) * N + s] = t.c01;
            o[(size_t)(2 * 4 + d) * N + s] = t.c10;
        }
    }
}

// proposals of one step of a group, one thread per cell (the proposers of the PatchMatch phase, lexp_kernels.cuh: pm_propose)
__global__ void lexp_gc_propose_kernel(const CallInfo* __restrict__ calls, int n, Plane4* __restrict__ planes, Plane4* planes_out,
                                       unsigned long long seed, const float4* cur_label, int W, int prop_kind, int prop_m, float min_disp, float max_disp) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (prop_kind) {
        const CallInfo ci = calls[i];
        const float4 g = pm_propose(ProposeArgs{seed, cur_label, W, prop_kind, prop_m, min_disp, max_disp}, ci.ux, ci.uy, ci.uw, ci.uh, ci.cell_id);
        planes[i] = Plane4{g.x, g.y, g.z, g.w};
    }
    if (planes_out) planes_out[i] = planes[i];
}

// initCurrentFast for any energy (FastGCStereo.h:101-113): `currentLabeling(unit) = label; ComputeUnaryPotential(.., currentCost(filterRegion), ..)`
// -- after the fused kernel has written the unary costs of the cells' labels into the proposalCost image, every cell's region takes them
// unconditionally.  One CTA per cell.  (The PatchMatch-phase kernel has this fused in, pm_mode 2.)
__global__ void lexp_gc_assign_kernel(const GcCell* __restrict__ cells, const Plane4* __restrict__ planes, const float* __restrict__ prop_cost,
                                      float* __restrict__ cur_cost, float4* __restrict__ cur_label, int W) {
    const GcCell c = cells[blockIdx.x];
    const Plane4 pl = planes[blockIdx.x];
    const float4 l1 = make_float4(pl.a, pl.b, pl.c, pl.v);
    const int N = c.w * c.h;
    for (int s = threadIdx.x; s < N; s += blockDim.x) {
        const size_t p = (size_t)(c.y + s / c.w) * W + (c.x + s % c.w);
        cur_cost[p] = prop_cost[p];
        cur_label[p] = l1;
    }
}

struct GcParams {
    const GcCell* cells;
    const Plane4* planes;            // [ncells] the proposal of every cell (label1)
    const float* prop_cost;          // float[H][W]: unary cost of the proposal on every cell's region (the fused kernel's image output)
    float* cur_cost;                 // currentCost_[mode]
    float4* cur_label;               // currentLabeling_[mode]
    const float4* coef;              // smoothness coefficients of this view
    float* scratch;                  // kGcWords planes of `scratch_nodes` floats / ints
    long long scratch_nodes;
    double* flows_out;               // [ncells] value of the move's minimum cut as BK reports it (optional)
    int* iters_out;                  // [ncells] push-relabel rounds used (optional, diagnostics)
    int* err_flag;                   // set to 2 when a move ran into max_rounds (the result is then not a minimum cut)
    int H, W;
    float lambda, th_smooth;
    int relabel_every;               // push / relabel rounds between two global relabelings
    int max_rounds;                  // safety bound on the total number of rounds
};

// ---- the expansion move: per-node steps, shared by the one-CTA-per-cell kernel and the phase kernels of large cells -------------------
//
// Graph (FastGCStereo.h:430-549): node s = pixel of the region with terminal weights
//     source S_s = currentCost(s) + sum_boundary cost00 + sum_{forward pairs (s, j)} C + sum_{forward pairs (i, s)} (D - C)
//     sink   T_s = proposalCost(s) + sum_boundary cost10
// and one arc s -> j of capacity max(0, B + C - D) per forward neighbour j inside the region (B = cost10, C = cost01, D = cost00 of the
// pair, StereoEnergy.h:441-449); boundary = neighbours outside the region but inside the image, which keep their label (:455-470).
// Only S - T shapes the cut; BK's flow value is sum_s min(S_s, T_s) + maxflow of what remains (see oracle/maxflow/graph.h).
//
// Minimum cut: synchronous push-relabel, deterministic (no floating-point atomics, relabels computed from the heights of the round's
// start: nothing depends on the order in which threads run): in a round every active node (excess > 0, finite
// height) first collects what its neighbours pushed to it in the previous round (push slots, double buffered), then pushes to the sink
// and along admissible arcs (height(v) == height(u) + 1) and records the amounts in its own push slots; after a barrier the nodes that
// still hold excess are relabelled.  Two neighbours never push along the same arc pair in the same round (the admissibility conditions
// exclude each other), so nobody else writes a node's residuals.  Every `relabel_every` rounds the heights are recomputed exactly
// (distance to the sink in the residual graph, by chaotic relaxation); nodes that cannot reach the sink get height infinity and stop
// being active.  The loop ends when no node is active right after such a global relabelling: the preflow is then maximum and
// height == infinity marks exactly the nodes from which the sink is unreachable = BK's SOURCE segment = the update mask.
struct GcView {       // the residual network of one cell inside the scratch planes
    GcCell c;
    int N;
    long long SN;
    float* ex;        // excess
    float* snk;       // residual capacity to the sink
    int* ht;          // height
    float* res;       // res[d * SN + s]: residual capacity of the arc s -> s + n_d
    float* pb;        // pb[(b * 8 + d) * SN + s]: amount s pushed along d in a round of parity b
    int* hq;          // height proposed by the node's last relabel; committed (max with ht) by its owner in the next push phase
};
__device__ __forceinline__ GcView gc_view(const GcParams& P, const GcCell c) {
    GcView V;
    V.c = c; V.N = c.w * c.h; V.SN = P.scratch_nodes;
    V.ex = P.scratch + c.node0;
    V.snk = P.scratch + V.SN + c.node0;
    V.ht = reinterpret_cast<int*>(P.scratch + 2 * V.SN) + c.node0;
    V.res = P.scratch + 3 * V.SN + c.node0;
    V.pb = P.scratch + 11 * V.SN + c.node0;
    V.hq = reinterpret_cast<int*>(P.scratch + 27 * V.SN) + c.node0;
    return V;
}

// Graph construction of node s.  The terminal weights are accumulated exactly as the reference's sequence of Graph::add_tweights calls does
// (BK keeps only the NET capacity tr = source - sink in float and moves the common part min(source, sink) into the flow value): first
// (currentCost, proposalCost) (:433), then the boundary terms in the reference's neighbour order (:455-470), then per forward direction
// GE, EG, LG, GG the pair in which the node is `j` (D - C) and the pair in which it is `i` (C) (:478-541; the pair loops run over (y, x)
// ascending, so a node is reached as `j` first).  With costs of 1e6 for invalid labels on both sides this keeps the small pairwise terms
// that a plain sum of the source weights in float would round away.  Returns BK's `flow += min(cap_source, cap_sink)` of the node.
__device__ __forceinline__ double gc_node_build(const GcParams& P, const GcView& V, const float4 l1, int s) {
    const GcCell& c = V.c;
    const int W = P.W, H = P.H;
    const float lambda = P.lambda, th = P.th_smooth;
    const long long SN = V.SN;
    const int x = s % c.w, y = s / c.w, X = c.x + x, Y = c.y + y;
    const size_t p = (size_t)Y * W + X;
    const float4 L0p = P.cur_label[p];
    const float4 cf = P.coef[p];
    float tr = 0.0f;
    double konst = 0.0;
    auto add_tweights = [&](float cap_source, float cap_sink) {   // Graph::add_tweights of the BK library
        if (tr > 0.0f) cap_source = __fadd_rn(cap_source, tr); else cap_sink = __fsub_rn(cap_sink, tr);
        konst += (double)(cap_source < cap_sink ? cap_source : cap_sink);
        tr = __fsub_rn(cap_source, cap_sink);
    };
    add_tweights(P.cur_cost[p], P.prop_cost[p]);                                                   // :433
    if (x == 0 || x == c.w - 1 || y == 0 || y == c.h - 1) {
#pragma unroll
        for (int k = 0; k < 8; k++) {   // the reference's neighbour order LE GE EL EG LL GL LG GG
            const int d = k == 0 ? 4 : k == 1 ? 0 : k == 2 ? 5 : k == 3 ? 1 : k == 4 ? 7 : k == 5 ? 6 : k == 6 ? 2 : 3;
            const int qx = x + gc_dx(d), qy = y + gc_dy(d), QX = X + gc_dx(d), QY = Y + gc_dy(d);
            if (qx >= 0 && qx < c.w && qy >= 0 && qy < c.h) continue;              // region.contains(pt)
            if (QX < 0 || QX >= W || QY < 0 || QY >= H) continue;                  // !imageDomain.contains(pt)
            const size_t q = (size_t)QY * W + QX;
            const float4 L0q = P.cur_label[q];                                     // the neighbour keeps its label
            const float co = d < 4 ? coef_of(cf, d) : coef_of(P.coef[q], d - 4);
            add_tweights(boundary_term(L0p, L0q, X, Y, QX, QY, co, lambda, th), boundary_term(l1, L0q, X, Y, QX, QY, co, lambda, th));   // :466-469
        }
    }
#pragma unroll
    for (int d = 0; d < 4; d++) {
        {   // this node is `j` of the pair whose `i` is the backward neighbour (:485, :500, :517, :534)
            const int qx = x - gc_dx(d), qy = y - gc_dy(d);
            if (qx >= 0 && qx < c.w && qy >= 0 && qy < c.h) {
                const size_t q = (size_t)(c.y + qy) * W + (c.x + qx);
                const PairTerms t = pair_terms(P.cur_label[q], L0p, l1, c.x + qx, c.y + qy, X, Y, true, coef_of(P.coef[q], d), lambda, th);
                add_tweights(__fsub_rn(t.c00, t.c01), 0.0f);
            }
        }
        float cap = 0.0f;
        const int qx = x + gc_dx(d), qy = y + gc_dy(d);
        if (qx >= 0 && qx < c.w && qy >= 0 && qy < c.h) {   // this node is `i` (:483-484)
            const size_t q = (size_t)(c.y + qy) * W + (c.x + qx);
            const PairTerms t = pair_terms(L0p, P.cur_label[q], l1, X, Y, c.x + qx, c.y + qy, true, coef_of(cf, d), lambda, th);
            cap = fmaxf(0.0f, __fsub_rn(__fadd_rn(t.c10, t.c01), t.c00));
            add_tweights(t.c01, 0.0f);
        }
        V.res[(size_t)d * SN + s] = cap;
        V.res[(size_t)(d + 4) * SN + s] = 0.0f;
    }
#pragma unroll
    for (int d = 0; d < 16; d++) V.pb[(size_t)d * SN + s] = 0.0f;
    V.ex[s] = tr > 0.0f ? tr : 0.0f;
    V.snk[s] = tr < 0.0f ? -tr : 0.0f;
    V.ht[s] = kGcInf;
    V.hq[s] = 0;
    return konst;
}
// start of a global relabelling: apply the pushes still pending in the neighbours' slots of parity `cur`, reset the height
__device__ __forceinline__ void gc_node_gather(const GcView& V, int s, int cur) {
    const GcCell& c = V.c;
    const int x = s % c.w, y = s / c.w;
    float e = V.ex[s];
#pragma unroll
    for (int d = 0; d < 8; d++) {
        const int qx = x + gc_dx(d), qy = y + gc_dy(d);
        if (qx >= 0 && qx < c.w && qy >= 0 && qy < c.h) {
            const float f = V.pb[(size_t)(cur * 8 + (d ^ 4)) * V.SN + (qy * c.w + qx)];
            if (f > 0.0f) { e += f; V.res[(size_t)d * V.SN + s] += f; }
        }
    }
    V.ex[s] = e;
    V.ht[s] = V.snk[s] > 0.0f ? 1 : kGcInf;
    V.hq[s] = 0;   // the exact distances replace whatever the last relabel proposed
}
__device__ __forceinline__ void gc_node_clear_slots(const GcView& V, int s, int cur) {
#pragma unroll
    for (int d = 0; d < 8; d++) V.pb[(size_t)(cur * 8 + d) * V.SN + s] = 0.0f;
}
// one pass of the chaotic relaxation h(v) = 1 + min over residual arcs v -> u of h(u) (converges to the BFS distances to the sink)
__device__ __forceinline__ int gc_node_relax(const GcView& V, int s) {
    const GcCell& c = V.c;
    const int hv = V.ht[s];
    if (hv == 1) return 0;
    const int x = s % c.w, y = s / c.w;
    int best = kGcInf;
#pragma unroll
    for (int d = 0; d < 8; d++) {
        const int qx = x + gc_dx(d), qy = y + gc_dy(d);
        if (qx >= 0 && qx < c.w && qy >= 0 && qy < c.h && V.res[(size_t)d * V.SN + s] > 0.0f) {
            const int hu = V.ht[qy * c.w + qx];
            if (hu < best) best = hu;
        }
    }
    if (best < kGcInf && best + 1 < hv) { V.ht[s] = best + 1; return 1; }
    return 0;
}
__device__ __forceinline__ int gc_node_active(const GcView& V, int s) { return V.ex[s] > 0.0f && V.ht[s] < kGcInf; }
// (A) collect the previous round's pushes, push to the sink and along admissible arcs; returns whether the node held excess
__device__ __forceinline__ int gc_node_push(const GcView& V, int s, int cur, double& to_sink) {
    const GcCell& c = V.c;
    const long long SN = V.SN;
    const int x = s % c.w, y = s / c.w;
    float e = V.ex[s];
    float rs[8];
    int hu[8];
#pragma unroll
    for (int d = 0; d < 8; d++) {
        const int qx = x + gc_dx(d), qy = y + gc_dy(d);
        rs[d] = 0.0f; hu[d] = kGcInf;
        if (qx >= 0 && qx < c.w && qy >= 0 && qy < c.h) {
            const int u = qy * c.w + qx;
            rs[d] = V.res[(size_t)d * SN + s];
            const float f = V.pb[(size_t)(cur * 8 + (d ^ 4)) * SN + u];
            if (f > 0.0f) { e += f; rs[d] += f; }
            hu[d] = max(V.ht[u], V.hq[u]);   // whether u has committed its proposal yet or not: the same value
        }
    }
    const int hv = max(V.ht[s], V.hq[s]);
    V.ht[s] = hv;                            // commit the height the last relabel proposed
    float out[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int busy = 0;
    if (e > 0.0f && hv < kGcInf) {
        busy = 1;
        const float cs = V.snk[s];
        if (cs > 0.0f) {   // a node with sink capacity has height 1: the arc to the sink is admissible
            const float f = e < cs ? e : cs;
            e -= f; V.snk[s] = cs - f; to_sink += (double)f;
        }
#pragma unroll
        for (int d = 0; d < 8; d++)
            if (e > 0.0f && rs[d] > 0.0f && hv == hu[d] + 1) {
                const float f = e < rs[d] ? e : rs[d];
                e -= f; rs[d] -= f; out[d] = f;
            }
    }
    V.ex[s] = e;
#pragma unroll
    for (int d = 0; d < 8; d++) {
        V.res[(size_t)d * SN + s] = rs[d];
        V.pb[(size_t)((cur ^ 1) * 8 + d) * SN + s] = out[d];
    }
    return busy;
}
// (B) relabel a node that still holds excess; an arc whose residual was created by a push of THIS round (still in the neighbour's push
// slot) counts as well.  The new height is only PROPOSED (hq): all relabels of a round are computed from the same committed heights, so
// the result does not depend on the order in which threads run; the owner commits it at the start of the next push phase, and readers
// take max(ht, hq) -- heights only grow, so a stale proposal never exceeds the committed height.
__device__ __forceinline__ void gc_node_relabel(const GcView& V, int s, int cur) {
    const GcCell& c = V.c;
    const int hv = V.ht[s];
    if (!(V.ex[s] > 0.0f && hv < kGcInf)) return;
    const int x = s % c.w, y = s / c.w;
    int best = V.snk[s] > 0.0f ? 0 : kGcInf;
#pragma unroll
    for (int d = 0; d < 8; d++) {
        const int qx = x + gc_dx(d), qy = y + gc_dy(d);
        if (qx >= 0 && qx < c.w && qy >= 0 && qy < c.h) {
            const int u = qy * c.w + qx;
            if (V.res[(size_t)d * V.SN + s] > 0.0f || V.pb[(size_t)((cur ^ 1) * 8 + (d ^ 4)) * V.SN + u] > 0.0f) {
                const int hq = V.ht[u];
                if (hq < best) best = hq;
            }
        }
    }
    const int hn = (best >= kGcInf || best + 1 > V.N + 1) ? kGcInf : best + 1;
    if (hn > hv) V.hq[s] = hn;   // proposed, not written to ht: every node of this phase sees the heights of the phase's start
}
// the move: `updateMask = what_segment(s) == SOURCE` (FastGCStereo.h:553-557), copyTo / setTo (:58-59); valid right after a global
// relabelling with no active node left: height == infinity <=> the sink is unreachable from the node
__device__ __forceinline__ void gc_node_apply(const GcParams& P, const GcView& V, const float4 l1, int s) {
    if (V.ht[s] >= kGcInf) {
        const int x = s % V.c.w, y = s / V.c.w;
        const size_t p = (size_t)(V.c.y + y) * P.W + (V.c.x + x);
        P.cur_cost[p] = P.prop_cost[p];
        P.cur_label[p] = l1;
    }
}

// The expansion move of one cell by ONE CTA (cells up to a few 10^4 nodes: layers 0 and 1): graph construction, minimum cut, copyTo / setTo.
// Thread t owns the nodes t, t + blockDim, ...; the phases are separated by __syncthreads().
__global__ void __launch_bounds__(1024) lexp_gc_move_kernel(const GcParams P) {
    __shared__ int s_flag[3];
    __shared__ double s_red[1024];
    const GcView V = gc_view(P, P.cells[blockIdx.x]);
    const Plane4 plv = P.planes[blockIdx.x];
    const float4 l1 = make_float4(plv.a, plv.b, plv.c, plv.v);
    const int N = V.N, T = blockDim.x, tid = threadIdx.x;

    double konst = 0.0;   // BK's `flow += min(cap_source, cap_sink)` over this thread's nodes
    for (int s = tid; s < N; s += T) konst += gc_node_build(P, V, l1, s);
    __syncthreads();

    double to_sink = 0.0;
    int cur = 0, rounds = 0;
    bool done = false;
    while (!done) {
        // ---- global relabelling: apply the pending pushes, then exact distances to the sink --------------------------------------
        for (int s = tid; s < N; s += T) gc_node_gather(V, s, cur);
        __syncthreads();
        for (int s = tid; s < N; s += T) gc_node_clear_slots(V, s, cur);
        for (;;) {
            if (tid == 0) s_flag[0] = 0;
            __syncthreads();
            int changed = 0;
            for (int s = tid; s < N; s += T) changed |= gc_node_relax(V, s);
            if (changed) s_flag[0] = 1;
            __syncthreads();
            const int any = s_flag[0];
            __syncthreads();
            if (!any) break;
        }
        // ---- push / relabel rounds ------------------------------------------------------------------------------------------------
        if (tid == 0) s_flag[1] = 0;
        __syncthreads();
        {
            int active = 0;
            for (int s = tid; s < N; s += T) active |= gc_node_active(V, s);
            if (active) s_flag[1] = 1;
        }
        __syncthreads();
        const int any_active = s_flag[1];
        __syncthreads();   // everybody has read the flag before it is reused below
        if (!any_active) { done = true; break; }
        if (rounds >= P.max_rounds) {   // never observed; bounded like every loop on the device: the host reports it (lexp_pm_get)
            if (tid == 0 && P.err_flag) atomicExch(P.err_flag, 2);
            done = true; break;
        }
        if (tid == 0) { s_flag[1] = 0; s_flag[2] = 0; }
        __syncthreads();
        for (int r = 0; r < P.relabel_every; r++, rounds++) {
            int busy = 0;
            for (int s = tid; s < N; s += T) busy |= gc_node_push(V, s, cur, to_sink);
            if (busy) s_flag[1 + (r & 1)] = 1;
            __syncthreads();
            const int any_busy = s_flag[1 + (r & 1)];
            if (tid == 0) s_flag[1 + ((r + 1) & 1)] = 0;   // next round's flag: last read before the previous round's second barrier
            for (int s = tid; s < N; s += T) gc_node_relabel(V, s, cur);
            __syncthreads();
            cur ^= 1;
            if (!any_busy) { rounds++; break; }
        }
    }

    for (int s = tid; s < N; s += T) gc_node_apply(P, V, l1, s);
    if (P.flows_out) {
        s_red[tid] = konst + to_sink;
        __syncthreads();
        if (tid == 0) {
            double f = 0.0;
            for (int i = 0; i < T; i++) f += s_red[i];
            P.flows_out[blockIdx.x] = f;
        }
    }
    if (P.iters_out && tid == 0) P.iters_out[blockIdx.x] = rounds;
}

// ---- large cells (layer 2: 3 * 10^5 nodes): the same steps as PHASE KERNELS over all SMs --------------------------------------------------
// One CTA per cell leaves 140 SMs idle when a group has 4-6 cells.  Here every phase of the loop above is a kernel of its own whose blocks
// of kGcPhaseThreads threads each own a run of consecutive nodes of one cell (block map built with the plan); the host issues the phases
// in the same order for all cells of the plan in lockstep and reads two flags back per decision (did a relaxation pass change a height?
// is any node active after the global relabelling?).  A cell that has finished (`done`) is skipped by every later phase; a round in which
// a cell has nothing to push is a no-op, so the result is identical to the one-CTA kernel's (same arithmetic, same rounds, same relabelling
// points) -- the emulator tests compare the two paths bit for bit.
constexpr int kGcPhaseThreads = 256;
struct GcBlock { int cell, first; };   // block b of a phase kernel: nodes [first, first + kGcPhaseThreads) of cell `cell`
struct GcPhaseCtl {
    const GcBlock* blocks;
    int* done;            // [ncells] the cell's minimum cut is complete
    int* active;          // [ncells] the cell has an active node (written by the `active` phase)
    int* g_flags;         // [0]: a relaxation pass changed a height; [1]: some cell is still active
    double* konst_part;   // [nblocks] BK's add_tweights constant, per block
    double* sink_part;    // [nblocks] flow pushed into the sink so far, per block
    int ncells;
};
enum { GC_PH_BUILD = 0, GC_PH_GATHER, GC_PH_CLEAR, GC_PH_RELAX, GC_PH_ACTIVE, GC_PH_PUSH, GC_PH_RELABEL, GC_PH_APPLY };

template <int PHASE>
__global__ void __launch_bounds__(kGcPhaseThreads) lexp_gc_phase_kernel(const GcParams P, const GcPhaseCtl C, int cur) {
    __shared__ double s_red[kGcPhaseThreads];
    const GcBlock b = C.blocks[blockIdx.x];
    if (PHASE != GC_PH_BUILD && PHASE != GC_PH_APPLY && C.done[b.cell]) return;
    const GcView V = gc_view(P, P.cells[b.cell]);
    const int s = b.first + threadIdx.x;
    const bool in = s < V.N;
    const Plane4 plv = P.planes[b.cell];
    const float4 l1 = make_float4(plv.a, plv.b, plv.c, plv.v);
    if (PHASE == GC_PH_BUILD || PHASE == GC_PH_PUSH) {
        double v = 0.0;
        if (PHASE == GC_PH_BUILD) { if (in) v = gc_node_build(P, V, l1, s); }
        else if (in) gc_node_push(V, s, cur, v);
        s_red[threadIdx.x] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
            double f = 0.0;
            for (int i = 0; i < kGcPhaseThreads; i++) f += s_red[i];
            if (PHASE == GC_PH_BUILD) { C.konst_part[blockIdx.x] = f; C.sink_part[blockIdx.x] = 0.0; }
            else if (f != 0.0) C.sink_part[blockIdx.x] += f;
        }
    } else if (in) {
        if (PHASE == GC_PH_GATHER) gc_node_gather(V, s, cur);
        if (PHASE == GC_PH_CLEAR) gc_node_clear_slots(V, s, cur);
        if (PHASE == GC_PH_RELAX) { if (gc_node_relax(V, s)) C.g_flags[0] = 1; }
        if (PHASE == GC_PH_ACTIVE) { if (gc_node_active(V, s)) C.active[b.cell] = 1; }
        if (PHASE == GC_PH_RELABEL) gc_node_relabel(V, s, cur);
        if (PHASE == GC_PH_APPLY) gc_node_apply(P, V, l1, s);
    }
}
// after the `active` phase: cells without an active node are done; g_flags[1] = some cell goes on.  One thread per cell.
__global__ void lexp_gc_phase_decide(const GcPhaseCtl C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C.ncells || C.done[i]) return;
    if (C.active[i]) { C.active[i] = 0; C.g_flags[1] = 1; }
    else C.done[i] = 1;
}
// flow of every cell = sum over its blocks (in block order) of the add_tweights constant and the flow into the sink
__global__ void lexp_gc_phase_flows(const GcPhaseCtl C, int nblocks, double* flows_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C.ncells) return;
    double f = 0.0;
    for (int b = 0; b < nblocks; b++) if (C.blocks[b].cell == i) f += C.konst_part[b] + C.sink_part[b];
    flows_out[i] = f;
}

}  // namespace lexp
