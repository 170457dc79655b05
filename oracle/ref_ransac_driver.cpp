// TEST INFRASTRUCTURE ONLY -- never part of the product path.
//
// C entry points around the reference's OWN RansacProposer (Proposer.h:155-312), compiled from its header where it lies over the
// mini cv:: layer of oracle/cvshim/ (see oracle/build_ref_ransac.py).  Nothing here restates RANSACPlane's control flow.  Three things
// are supplied, and substituted inside the reference's header only:
//   * cv::solve(DECOMP_SVD): the shim's stub refuses it.  Here it is the device's contract (DESIGN.md section 3f): the minimum-norm
//     least-squares solution in double with the exact rank of the integer rows, full-rank systems centred on the unit region, A^T b as
//     a correctly rounded sum, a fixed cyclic Jacobi sequence -- more accurate than OpenCV's float Jacobi SVD, which cannot be reproduced.
//   * cv::countNonZero: the shim's, recording every count (no_i, and no after a refit), so the per-sample trace can be compared.
//   * rand(): std::random_shuffle draws from the process-global rand().  This library defines its own rand() and is linked with
//     -Bsymbolic, so the shuffle inside it calls this one: it returns the swap indices that make the first three entries of the
//     permutation the injected triple of each sample.  ref_ransac_shuffle_check shows that the interposition is in effect.
// Output: oracle/_ref/liblexp_ref_ransac.so.
#include <opencv2/opencv.hpp>
#include "Utilities.hpp"
#include "Plane.h"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <numeric>
#include <vector>

namespace {
std::vector<int> g_tri;          // injected triples, 3 per sample
size_t g_sample = 0;             // samples started so far
int g_n = 0, g_step = 0;         // length of the permutation being shuffled; rand() calls so far within it
int g_j1 = 0, g_j2 = 0;
int g_cx = 0, g_cy = 0;          // integer centre of the unit region (the solve centres full-rank systems on it)
std::vector<int> g_counts, g_sample_of_count;

void start_sample() {
    const int* t = g_sample < g_tri.size() / 3 ? &g_tri[3 * g_sample] : nullptr;
    g_sample++;
    g_j1 = 1; g_j2 = 2;
    if (!t) return;
    for (int j1 = 0; j1 < 2; j1++)       // steps 1 and 2 of the shuffle arrange {0, 1, 2}; steps i = t_p >= 3 bring t_p to position p
        for (int j2 = 0; j2 < 3; j2++) {
            int v[3] = {0, 1, 2};
            std::swap(v[1], v[j1]);
            std::swap(v[2], v[j2]);
            bool ok = true;
            for (int p = 0; p < 3; p++) ok = ok && (t[p] >= 3 || v[p] == t[p]);
            if (ok) { g_j1 = j1; g_j2 = j2; return; }
        }
}

// Python's math.fsum (Shewchuk's partials, then the correctly rounded total) for finite values
double fsum(const std::vector<double>& xs) {
    std::vector<double> p;
    for (double x : xs) {
        size_t i = 0;
        for (size_t k = 0; k < p.size(); k++) {
            double y = p[k];
            if (std::fabs(x) < std::fabs(y)) std::swap(x, y);
            const double hi = x + y, lo = y - (hi - x);
            if (lo != 0.0) p[i++] = lo;
            x = hi;
        }
        p.resize(i);
        p.push_back(x);
    }
    size_t n = p.size();
    double hi = 0.0;
    if (n > 0) {
        hi = p[--n];
        double lo = 0.0;
        while (n > 0) {
            const double x = hi, y = p[--n];
            hi = x + y;
            lo = y - (hi - x);
            if (lo != 0.0) break;
        }
        if (n > 0 && ((lo < 0.0 && p[n - 1] < 0.0) || (lo > 0.0 && p[n - 1] > 0.0))) {
            const double y = lo * 2.0, x = hi + y;
            if (y == x - hi) hi = x;
        }
    }
    return hi;
}

int gram_rank(const long long G[6]) {   // xx, xy, yy, x, y, n
    if (G[5] == 0) return 0;
    const __int128 sxx = (__int128)G[5] * G[0] - (__int128)G[3] * G[3], syy = (__int128)G[5] * G[2] - (__int128)G[4] * G[4];
    const __int128 sxy = (__int128)G[5] * G[1] - (__int128)G[3] * G[4];
    if (sxx == 0 && syy == 0) return 1;
    return sxx * syy == sxy * sxy ? 2 : 3;
}

void minnorm(const long long G[6], const double g[3], int rank, double N[3]) {   // compiled with -ffp-contract=off
    double a[3][3] = {{(double)G[0], (double)G[1], (double)G[3]}, {(double)G[1], (double)G[2], (double)G[4]}, {(double)G[3], (double)G[4], (double)G[5]}};
    double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 8; sweep++)
        for (int pq = 0; pq < 3; pq++) {
            const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2, r = 3 - p - q;
            const double apq = a[p][q];
            if (apq == 0.0) continue;
            const double tau = (a[q][q] - a[p][p]) / (2.0 * apq);
            double t = 1.0 / (std::fabs(tau) + std::sqrt(1.0 + tau * tau));
            if (tau < 0.0) t = -t;
            const double c = 1.0 / std::sqrt(1.0 + t * t), s = t * c;
            a[p][p] = a[p][p] - t * apq;
            a[q][q] = a[q][q] + t * apq;
            a[p][q] = a[q][p] = 0.0;
            const double arp = a[r][p], arq = a[r][q];
            a[r][p] = a[p][r] = c * arp - s * arq;
            a[r][q] = a[q][r] = s * arp + c * arq;
            for (int k = 0; k < 3; k++) {
                const double vkp = V[k][p], vkq = V[k][q];
                V[k][p] = c * vkp - s * vkq;
                V[k][q] = s * vkp + c * vkq;
            }
        }
    bool keep[3] = {true, true, true};
    for (int d = rank; d < 3; d++) {
        int m = -1;
        for (int j = 0; j < 3; j++) if (keep[j] && (m < 0 || a[j][j] < a[m][m])) m = j;
        keep[m] = false;
    }
    N[0] = N[1] = N[2] = 0.0;
    for (int i = 0; i < 3; i++)
        if (keep[i]) {
            const double d = (V[0][i] * g[0] + V[1][i] * g[1]) + V[2][i] * g[2];
            const double w = d / a[i][i];
            for (int k = 0; k < 3; k++) N[k] = N[k] + V[k][i] * w;
        }
}
}  // namespace

extern "C" int rand(void) throw() {   // the shuffle's swap index of step i = g_step: j = rand() % (i + 1)
    if (g_step == 0) start_sample();
    const int i = ++g_step;
    if (g_step >= g_n - 1) g_step = 0;
    const size_t s = g_sample - 1;
    if (s < g_tri.size() / 3) {
        const int* t = &g_tri[3 * s];
        if (i == 1) return g_j1;
        if (i == 2) return g_j2;
        for (int p = 0; p < 3; p++) if (t[p] == i) return p;
    }
    return i;
}

namespace cv {
inline bool lexp_pin_solve(const Mat& A, const Mat& b, const OutputArray& dst, int flags) {
    if (flags != DECOMP_SVD || A.type() != CV_32FC1 || b.type() != CV_32FC1 || A.cols != 3 || b.rows != A.rows) shim_fail("solve: only the RANSAC systems");
    long long G[6] = {0, 0, 0, 0, 0, 0}, Gc[6] = {0, 0, 0, 0, 0, 0};
    std::vector<double> px, py, pb, qx, qy;
    bool finite = true;
    for (int r = 0; r < A.rows; r++) {   // rows (x, y, 1), or zero rows (Proposer.h:200-213 leaves the unused rows of A at zero)
        const long long x = (long long)A.at<float>(r, 0), y = (long long)A.at<float>(r, 1), w = (long long)A.at<float>(r, 2);
        const double bv = (double)b.at<float>(r, 0);
        finite = finite && std::isfinite(bv);
        G[0] += x * x; G[1] += x * y; G[2] += y * y; G[3] += x * w; G[4] += y * w; G[5] += w * w;
        const long long xc = x - g_cx * w, yc = y - g_cy * w;
        Gc[0] += xc * xc; Gc[1] += xc * yc; Gc[2] += yc * yc; Gc[3] += xc * w; Gc[4] += yc * w; Gc[5] += w * w;
        px.push_back((double)x * bv); py.push_back((double)y * bv); pb.push_back((double)w * bv);
        qx.push_back((double)xc * bv); qy.push_back((double)yc * bv);
    }
    Mat N(3, 1, CV_32FC1);
    if (!finite) {   // never an inlier of anything (the oracle returns NaN too)
        for (int k = 0; k < 3; k++) N.at<float>(k, 0) = NAN;
        dst.assign(N);
        return true;
    }
    const int rank = gram_rank(G);
    double out[3];
    if (rank == 3) {
        const double g[3] = {fsum(qx), fsum(qy), fsum(pb)};
        minnorm(Gc, g, 3, out);
        out[2] = out[2] - (out[0] * (double)g_cx + out[1] * (double)g_cy);
    } else {
        const double g[3] = {fsum(px), fsum(py), fsum(pb)};
        minnorm(G, g, rank, out);
    }
    for (int k = 0; k < 3; k++) N.at<float>(k, 0) = (float)out[k];
    dst.assign(N);
    return true;
}
inline int lexp_pin_count_nonzero(const Mat& a) {
    const int n = countNonZero(a);
    g_counts.push_back(n);
    g_sample_of_count.push_back((int)g_sample - 1);
    return n;
}
}  // namespace cv
#define solve lexp_pin_solve
#define countNonZero lexp_pin_count_nonzero
#include "Proposer.h"
#undef solve
#undef countNonZero

namespace {
struct RansacProbe : RansacProposer {
    using RansacProposer::RansacProposer;
    using RansacProposer::computeSampleCount;
};
void inject(const int* triples, int n_triples, int n) {
    g_tri.assign(triples, triples + 3 * (size_t)n_triples);
    g_sample = 0; g_step = 0; g_n = n;
    g_counts.clear(); g_sample_of_count.clear();
}
}  // namespace

extern "C" {

// RansacProposer(1): startIterations(labeling, unit, 0), then getNextProposal, with the samples' triples injected.  labeling: float
// [H][W][4].  Outputs: the plane, the number of samples drawn, and per count (every countNonZero of RANSACPlane, in order) its value
// and the sample it belongs to.  Returns the number of counts, or -1 if cap is too small.
__attribute__((visibility("default"))) int ref_ransac_run(const float* labeling, int H, int W, int ux, int uy, int uw, int uh, const int* triples,
                                                          int n_triples, float* plane_out, int* n_samples, int* counts, int* sample_of_count, int cap) {
    cv::Mat lab(H, W, CV_32FC4, const_cast<float*>(labeling));
    inject(triples, n_triples, uw * uh);
    g_cx = ux + uw / 2; g_cy = uy + uh / 2;
    RansacProposer proto(1);
    IProposer* prop = proto.createInstance();
    prop->startIterations(lab, cv::Rect(ux, uy, uw, uh), 0);
    const Plane p = prop->getNextProposal();
    delete prop;
    plane_out[0] = p.a; plane_out[1] = p.b; plane_out[2] = p.c; plane_out[3] = p.v;
    *n_samples = (int)g_sample;
    if ((int)g_counts.size() > cap) return -1;
    for (size_t i = 0; i < g_counts.size(); i++) { counts[i] = g_counts[i]; sample_of_count[i] = g_sample_of_count[i]; }
    return (int)g_counts.size();
}

__attribute__((visibility("default"))) int ref_ransac_sample_count(int ni, int pt_num) {
    RansacProbe p(1);
    return p.computeSampleCount(ni, pt_num, 3, 0.95f);
}

// self-check of the interposition: std::random_shuffle of 0..n-1 (the reference's randperm) with one injected triple
__attribute__((visibility("default"))) void ref_ransac_shuffle_check(int n, const int* triple, int* first3) {
    inject(triple, 1, n);
    std::vector<int> v(n);
    std::iota(v.begin(), v.end(), 0);
    std::random_shuffle(v.begin(), v.end());
    for (int i = 0; i < 3; i++) first3[i] = v[i];
}

}  // extern "C"
