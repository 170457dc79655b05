/* CPU oracle (plain C + OpenMP) for the LocalExpStereo unary-cost hot path.
 * TEST / BASELINE INFRASTRUCTURE ONLY -- never linked into the product library.
 *
 * Independent restatement (double-precision guided filter, running-sum box
 * filter, same loop structure as the reference) of:
 *   CostVolumeEnergy::ComputeUnaryPotential[WithoutCheck]  CostVolumeEnergy.h:55-98,169-183
 *   GuidedImageFilter<double> ctor / filter_raw / filter    GuidedFilter.h:58-102,142-266
 *   FastGuidedImageFilter::createSubregionFilter            GuidedFilter.h:301-326
 *   StereoEnergy::IsValiLabel                               StereoEnergy.h:560-610
 * (paths relative to /root/reference/LocalExpansionStereo/).
 *
 * PARITY STATUS: pinned by the reference's own code -- tests/test_ref_pin.py holds this file (and the numpy oracle)
 * against oracle/_ref/liblexp_ref.so, the reference's CostVolumeEnergy / FastGuidedImageFilter<double> classes compiled
 * from its headers (oracle/build_ref.py), and against the reference-minted tests/golden/ vectors.  It is also one of the
 * two timed CPU baselines of bench.py (kind "port"; the other is the compiled reference itself, kind "reference"): one
 * OpenMP thread per cell of a batch, like the reference's `#pragma omp parallel for` over the cells of a disjoint group
 * (FastGCStereo.h:30).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define COST_FOR_INVALID 1000000.0f /* StereoEnergy.h:45 */

typedef struct {
    int H, W, D, R;
    double eps;
    float th_col, min_disp, max_disp;
    const float* vol[2];      /* borrowed: float[D][H][W] */
    double* I[2][3];          /* realI channels            GuidedFilter.h:62-67 */
    double* mean[2][3];       /* mean_I_{r,g,b}            GuidedFilter.h:70-72 */
    double* inv[2][6];        /* inv{rr,rg,rb,gg,gb,bb}    GuidedFilter.h:87-101 */
} oracle_ctx;

/* cv::boxFilter(ksize 2R+1, normalize=false, BORDER_CONSTANT) on a w x h double
 * image with row stride `ss` (GuidedFilter.h:40-45): running row sums, then running
 * column sums.  `tmp` holds w*h doubles. */
static void box_sum(const double* src, int ss, double* dst, int w, int h, int R, double* tmp, double* acc) {
    for (int y = 0; y < h; y++) {
        const double* s = src + (size_t)y * ss;
        double* t = tmp + (size_t)y * w;
        double run = 0;
        for (int x = 0; x < R && x < w; x++) run += s[x];
        for (int x = 0; x < w; x++) {
            if (x + R < w) run += s[x + R];
            if (x - R - 1 >= 0) run -= s[x - R - 1];
            t[x] = run;
        }
    }
    /* column running sums, row-major friendly */
    for (int x = 0; x < w; x++) acc[x] = 0;
    for (int y = 0; y < R && y < h; y++)
        for (int x = 0; x < w; x++) acc[x] += tmp[(size_t)y * w + x];
    for (int y = 0; y < h; y++) {
        if (y + R < h)
            for (int x = 0; x < w; x++) acc[x] += tmp[(size_t)(y + R) * w + x];
        if (y - R - 1 >= 0)
            for (int x = 0; x < w; x++) acc[x] -= tmp[(size_t)(y - R - 1) * w + x];
        memcpy(dst + (size_t)y * w, acc, (size_t)w * sizeof(double));
    }
}

void* oracle_create(int H, int W, int D, int windR, double eps, float th_col, float min_disp, float max_disp) {
    oracle_ctx* c = (oracle_ctx*)calloc(1, sizeof(oracle_ctx));
    c->H = H; c->W = W; c->D = D; c->R = windR / 2; /* CostVolumeEnergy.h:30 */
    c->eps = eps; c->th_col = th_col; c->min_disp = min_disp; c->max_disp = max_disp;
    return c;
}

void oracle_destroy(void* p) {
    oracle_ctx* c = (oracle_ctx*)p;
    if (!c) return;
    for (int m = 0; m < 2; m++) {
        for (int k = 0; k < 3; k++) { free(c->I[m][k]); free(c->mean[m][k]); }
        for (int k = 0; k < 6; k++) free(c->inv[m][k]);
    }
    free(c);
}

void oracle_set_volume(void* p, int mode, const float* vol) { ((oracle_ctx*)p)->vol[mode] = vol; }

/* GuidedImageFilter<double>(I, R, eps, 1/255) constructor, GuidedFilter.h:58-102. bgr = uint8[H][W][3]. */
void oracle_set_image(void* p, int mode, const uint8_t* bgr) {
    oracle_ctx* c = (oracle_ctx*)p;
    const int H = c->H, W = c->W, R = c->R;
    const size_t n = (size_t)H * W;
    double *N = (double*)malloc(n * 8), *tmp = (double*)malloc(n * 8), *prod = (double*)malloc(n * 8), *acc = (double*)malloc((size_t)W * 8);
    double* var[6];
    for (int k = 0; k < 3; k++) {
        free(c->I[mode][k]); free(c->mean[mode][k]);
        c->I[mode][k] = (double*)malloc(n * 8);
        c->mean[mode][k] = (double*)malloc(n * 8);
        for (size_t i = 0; i < n; i++) c->I[mode][k][i] = (double)bgr[i * 3 + k] * (1.0 / 255); /* :62-65 */
    }
    for (size_t i = 0; i < n; i++) prod[i] = 1.0;
    box_sum(prod, W, N, W, H, R, tmp, acc); /* :69 */
    for (int k = 0; k < 3; k++) {
        box_sum(c->I[mode][k], W, c->mean[mode][k], W, H, R, tmp, acc);
        for (size_t i = 0; i < n; i++) c->mean[mode][k][i] /= N[i]; /* :70-72 */
    }
    static const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {0, 1, 2, 1, 2, 2}; /* rr rg rb gg gb bb */
    for (int k = 0; k < 6; k++) {
        var[k] = (double*)malloc(n * 8);
        const double *A = c->I[mode][pa[k]], *B = c->I[mode][pb[k]];
        const double *mA = c->mean[mode][pa[k]], *mB = c->mean[mode][pb[k]];
        for (size_t i = 0; i < n; i++) prod[i] = A[i] * B[i];
        box_sum(prod, W, var[k], W, H, R, tmp, acc);
        const double e = (pa[k] == pb[k]) ? c->eps : 0.0;
        for (size_t i = 0; i < n; i++) var[k][i] = var[k][i] / N[i] - mA[i] * mB[i] + e; /* :79-84 */
    }
    for (int k = 0; k < 6; k++) { free(c->inv[mode][k]); c->inv[mode][k] = (double*)malloc(n * 8); }
    for (size_t i = 0; i < n; i++) {
        const double rr = var[0][i], rg = var[1][i], rb = var[2][i], gg = var[3][i], gb = var[4][i], bb = var[5][i];
        double irr = gg * bb - gb * gb, irg = gb * rb - rg * bb, irb = rg * gb - gg * rb; /* :87-92 */
        double igg = rr * bb - rb * rb, igb = rb * rg - rr * gb, ibb = rr * gg - rg * rg;
        const double det = irr * rr + irg * rg + irb * rb; /* :94 */
        c->inv[mode][0][i] = irr / det; c->inv[mode][1][i] = irg / det; c->inv[mode][2][i] = irb / det;
        c->inv[mode][3][i] = igg / det; c->inv[mode][4][i] = igb / det; c->inv[mode][5][i] = ibb / det;
    }
    for (int k = 0; k < 6; k++) free(var[k]);
    free(N); free(tmp); free(prod); free(acc);
}

/* export the 9 float statistics planes [mean r,g,b, inv rr,rg,rb,gg,gb,bb] (for cross-checks) */
void oracle_get_stats(void* p, int mode, float* out9) {
    oracle_ctx* c = (oracle_ctx*)p;
    const size_t n = (size_t)c->H * c->W;
    for (int k = 0; k < 3; k++) for (size_t i = 0; i < n; i++) out9[k * n + i] = (float)c->mean[mode][k][i];
    for (int k = 0; k < 6; k++) for (size_t i = 0; i < n; i++) out9[(3 + k) * n + i] = (float)c->inv[mode][k][i];
}

/* HOT LOOP 1: CostVolumeEnergy.h:69-98 (interpolate == 1). raw = float[fh][fw]. */
void oracle_sample(void* p, int mode, int fx, int fy, int fw, int fh, const float* plane, float* raw) {
    oracle_ctx* c = (oracle_ctx*)p;
    const int D = c->D, H = c->H, W = c->W;
    const float MIN = c->min_disp, MAX = c->max_disp;
    const int D0 = (int)(-MIN);
    const float* vol = c->vol[mode];
    const size_t HW = (size_t)H * W;
    const float a = plane[0], b = plane[1], cc = plane[2];
    for (int y = fy; y < fy + fh; y++) {
        float* pC = raw + (size_t)(y - fy) * fw;
        volatile float by = b * (float)y; /* volatile: forbid FMA contraction */
        const float d_base = by + cc;
        for (int x = fx; x < fx + fw; x++) {
            volatile float ax = a * (float)x;
            const float d = ax + d_base;
            float C;
            if (d < MIN) C = vol[(size_t)y * W + x];
            else if (d >= MAX) C = vol[(size_t)(D - 1) * HW + (size_t)y * W + x];
            else if (isnan(d) || isinf(d)) C = COST_FOR_INVALID;
            else {
                const int d0 = (int)d + D0, d1 = d0 + 1;
                const float f1 = d - floorf(d), f0 = 1.0f - f1;
                if (d1 >= D || d0 < 0) C = COST_FOR_INVALID;
                else {
                    volatile float t0 = f0 * vol[(size_t)d0 * HW + (size_t)y * W + x];
                    volatile float t1 = f1 * vol[(size_t)d1 * HW + (size_t)y * W + x];
                    C = t0 + t1;
                }
            }
            pC[x - fx] = (c->th_col < C) ? c->th_col : C; /* std::min(C, th_col) */
        }
    }
}

static inline int valid_ds(float ds, float a5, float b5, float MIN, float MAX) {
    float d;
    return ds >= MIN && ds <= MAX && ((d = ds + a5 + b5) >= MIN) && d <= MAX && ((d = ds + a5 - b5) >= MIN) && d <= MAX &&
           ((d = ds - a5 + b5) >= MIN) && d <= MAX && ((d = ds - a5 - b5) >= MIN) && d <= MAX;
}

/* One call of ComputeUnaryPotential[WithoutCheck].  out = float[th][tw] (row stride out_stride floats). */
/* scratch of one worker thread: reused across calls (a malloc/free per call serialises the OpenMP threads in the
 * allocator and makes the baseline scale negatively) */
typedef struct { size_t cap; float* raw; double* buf; } oracle_scratch;
static void scratch_reserve(oracle_scratch* s, size_t n, size_t w) {
    const size_t need = n + w;
    if (need <= s->cap) return;
    free(s->raw); free(s->buf);
    s->raw = (float*)malloc(n * sizeof(float));
    s->buf = (double*)malloc((n * 10 + w) * sizeof(double));
    s->cap = need;
}

static void oracle_unary_s(void* p, int mode, const int* frect, const int* trect, const float* plane, float* out, int out_stride,
                           int with_check, oracle_scratch* sc) {
    oracle_ctx* c = (oracle_ctx*)p;
    const int W = c->W, R = c->R;
    const int fx = frect[0], fy = frect[1], fw = frect[2], fh = frect[3];
    const int tx = trect[0], ty = trect[1], tw = trect[2], th = trect[3];
    const size_t n = (size_t)fw * fh;
    scratch_reserve(sc, n, (size_t)fw);
    float* raw = sc->raw;
    double* buf = sc->buf;
    double* acc = buf + n * 10;
    double *P = buf, *Br = buf + n, *Bg = buf + 2 * n, *Bb = buf + 3 * n, *Ar = buf + 4 * n, *Ag = buf + 5 * n,
           *Ab = buf + 6 * n, *Bq = buf + 7 * n, *tmp = buf + 8 * n, *N = buf + 9 * n;
    oracle_sample(p, mode, fx, fy, fw, fh, plane, raw);
    /* N = boxfilter(ones(rect.size()))  GuidedFilter.h:324 */
    for (size_t i = 0; i < n; i++) Bq[i] = 1.0;
    box_sum(Bq, fw, N, fw, fh, R, tmp, acc);
    const double *Ir = c->I[mode][0], *Ig = c->I[mode][1], *Ib = c->I[mode][2];
    for (int y = 0; y < fh; y++)
        for (int x = 0; x < fw; x++) { /* :151-169 */
            const size_t i = (size_t)y * fw + x, g = (size_t)(fy + y) * W + fx + x;
            const double vp = (double)raw[i];
            P[i] = vp; Br[i] = Ir[g] * vp; Bg[i] = Ig[g] * vp; Bb[i] = Ib[g] * vp;
        }
    box_sum(P, fw, Bq, fw, fh, R, tmp, acc); memcpy(P, Bq, n * 8);   /* :145 */
    box_sum(Br, fw, Bq, fw, fh, R, tmp, acc); memcpy(Br, Bq, n * 8); /* :170-172 */
    box_sum(Bg, fw, Bq, fw, fh, R, tmp, acc); memcpy(Bg, Bq, n * 8);
    box_sum(Bb, fw, Bq, fw, fh, R, tmp, acc); memcpy(Bb, Bq, n * 8);
    for (int y = 0; y < fh; y++)
        for (int x = 0; x < fw; x++) { /* :180-222 */
            const size_t i = (size_t)y * fw + x, g = (size_t)(fy + y) * W + fx + x;
            const double nn = N[i], mp = P[i] / nn;
            const double mIr = c->mean[mode][0][g], mIg = c->mean[mode][1][g], mIb = c->mean[mode][2][g];
            const double cr = Br[i] / nn - mIr * mp, cg = Bg[i] / nn - mIg * mp, cb = Bb[i] / nn - mIb * mp;
            const double *v0 = c->inv[mode][0], *v1 = c->inv[mode][1], *v2 = c->inv[mode][2], *v3 = c->inv[mode][3],
                         *v4 = c->inv[mode][4], *v5 = c->inv[mode][5];
            const double ar = v0[g] * cr + v1[g] * cg + v2[g] * cb;
            const double ag = v1[g] * cr + v3[g] * cg + v4[g] * cb;
            const double ab = v2[g] * cr + v4[g] * cg + v5[g] * cb;
            Ar[i] = ar; Ag[i] = ag; Ab[i] = ab;
            P[i] = mp - ar * mIr - ag * mIg - ab * mIb; /* b, :220 */
        }
    box_sum(Ar, fw, Bq, fw, fh, R, tmp, acc); memcpy(Ar, Bq, n * 8); /* :224-227 */
    box_sum(Ag, fw, Bq, fw, fh, R, tmp, acc); memcpy(Ag, Bq, n * 8);
    box_sum(Ab, fw, Bq, fw, fh, R, tmp, acc); memcpy(Ab, Bq, n * 8);
    box_sum(P, fw, Bq, fw, fh, R, tmp, acc);
    const float MIN = c->min_disp, MAX = c->max_disp;
    const float a = plane[0], b = plane[1], cc = plane[2], v = plane[3];
    const float a5 = a * 5, b5 = b * 5;
    for (int y = ty; y < ty + th; y++)
        for (int x = tx; x < tx + tw; x++) {
            const size_t i = (size_t)(y - fy) * fw + (x - fx), g = (size_t)y * W + x;
            const double q = (Bq[i] + Ar[i] * Ir[g] + Ag[i] * Ig[g] + Ab[i] * Ib[g]) / N[i]; /* :243 */
            float r = (float)q;                                                              /* :260-263 */
            if (with_check) { /* StereoEnergy.h:577-610 */
                float ds;
                if (tw == 1 && th == 1) {
                    volatile float t0 = a * (float)x, t1 = b * (float)y;
                    volatile float t2 = t0 + t1;
                    ds = t2 + cc;
                } else {
                    volatile float t0 = (float)x * a, t1 = (float)y * b, t2 = cc * 1.0f, t3 = 0.0f * v;
                    volatile float s = t0 + t1;
                    s = s + t2;
                    s = s + t3;
                    ds = s;
                }
                if (!valid_ds(ds, a5, b5, MIN, MAX)) r = COST_FOR_INVALID; /* CostVolumeEnergy.h:180-182 */
            }
            out[(size_t)(y - ty) * out_stride + (x - tx)] = r;
        }
}

void oracle_unary(void* p, int mode, const int* frect, const int* trect, const float* plane, float* out, int out_stride,
                  int with_check) {
    oracle_scratch sc = {0, NULL, NULL};
    oracle_unary_s(p, mode, frect, trect, plane, out, out_stride, with_check, &sc);
    free(sc.raw); free(sc.buf);
}

/* A batch = the cells of one (layer, group, step): one OpenMP thread per cell (FastGCStereo.h:30-49).
 * out_base is an H x W float image; every call writes costs(targetRect) in image coordinates. */
void oracle_unary_batch(void* p, int mode, int ncalls, const int* frects, const int* trects, const float* planes,
                        float* out_base, int with_check, int nthreads) {
    oracle_ctx* c = (oracle_ctx*)p;
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel
    {
        /* the scratch outlives the call (libgomp keeps its worker threads): allocating ~1 MB per thread per call means an
         * mmap/munmap pair each, whose TLB shootdowns serialise the threads -- measured as NEGATIVE scaling in a VM */
        static __thread oracle_scratch sc = {0, NULL, NULL};
#pragma omp for schedule(dynamic, 1)
        for (int i = 0; i < ncalls; i++) {
            const int* t = trects + 4 * i;
            oracle_unary_s(p, mode, frects + 4 * i, t, planes + 4 * i, out_base + (size_t)t[1] * c->W + t[0], c->W, with_check, &sc);
        }
    }
}

/* ------------------------------------------------------------------------------------------------------------------
 * The reference's two other aggregation filters of CostVolumeEnergy (oracle/filter_oracle.py restates them in numpy):
 *   filter 1, BilateralFilter::filter (GuidedFilter.h:329-373, filterName "BL"):
 *       q(x) = sum over y in (x +- windR) & filterRect of p(y) exp(-(|B(y)-B(x)| + |G(y)-G(x)| + |R(y)-R(x)|) / sig2),
 *     the 8-bit BGR guide of the view, the raw costs p of oracle_sample, not normalised;
 *   filter 2, filterName "": the raw cost itself (CostVolumeEnergy.h:169-171).
 * Weights exp(-s / sig2) in FP64 from a table over the integer channel sum s (0 .. 765: exact), window sums in FP64, the
 * window walked row by row from the top and each row from the left (the numpy oracle's order).  out_q / out_scale are
 * H x W double images: every call writes q and sum w |p| (|q| for "") on its targetRect; with_check sets both to
 * COST_FOR_INVALID where IsValiLabel fails (CostVolumeEnergy.h:176-182).  One OpenMP thread per cell.
 * ------------------------------------------------------------------------------------------------------------------ */
#define ORACLE_FILTER_BILATERAL 1 /* LEXP_FILTER_BILATERAL */
#define ORACLE_FILTER_NONE 2      /* LEXP_FILTER_NONE */

/* StereoEnergy::IsValiLabel at (x, y) of targetRect (tw x th): the float arithmetic of oracle_unary_s's check */
static int label_valid(const float* plane, int x, int y, int tw, int th, float MIN, float MAX) {
    const float a = plane[0], b = plane[1], cc = plane[2], v = plane[3];
    const float a5 = a * 5, b5 = b * 5;
    float ds;
    if (tw == 1 && th == 1) {
        volatile float t0 = a * (float)x, t1 = b * (float)y;
        volatile float t2 = t0 + t1;
        ds = t2 + cc;
    } else {
        volatile float t0 = (float)x * a, t1 = (float)y * b, t2 = cc * 1.0f, t3 = 0.0f * v;
        volatile float s = t0 + t1;
        s = s + t2;
        s = s + t3;
        ds = s;
    }
    return valid_ds(ds, a5, b5, MIN, MAX);
}

typedef struct { size_t cap; float* raw; int* guide; } filter_scratch;

static void oracle_filter_unary_s(oracle_ctx* c, int mode, const int* frect, const int* trect, const float* plane, double* out_q,
                                  double* out_scale, int with_check, int filter, int R, const double* wtab, filter_scratch* sc) {
    const int W = c->W;
    const int fx = frect[0], fy = frect[1], fw = frect[2], fh = frect[3];
    const int tx = trect[0], ty = trect[1], tw = trect[2], th = trect[3];
    const size_t n = (size_t)fw * fh;
    if (n > sc->cap) {
        free(sc->raw); free(sc->guide);
        sc->raw = (float*)malloc(n * sizeof(float));
        sc->guide = (int*)malloc(n * 3 * sizeof(int));
        sc->cap = n;
    }
    float* raw = sc->raw;
    int* G = sc->guide;
    oracle_sample(c, mode, fx, fy, fw, fh, plane, raw);
    if (filter == ORACLE_FILTER_BILATERAL)   /* the 8-bit guide back from realI = B / 255 (exact after rounding) */
        for (int y = 0; y < fh; y++)
            for (int x = 0; x < fw; x++) {
                const size_t i = (size_t)y * fw + x, g = (size_t)(fy + y) * W + fx + x;
                for (int k = 0; k < 3; k++) G[i * 3 + k] = (int)lround(c->I[mode][k][g] * 255.0);
            }
    for (int y = ty; y < ty + th; y++)
        for (int x = tx; x < tx + tw; x++) {
            const size_t o = (size_t)y * W + x;
            const size_t ci = (size_t)(y - fy) * fw + (x - fx);
            double q, s;
            if (filter == ORACLE_FILTER_BILATERAL) {
                const int* g0 = G + ci * 3;
                const int y0 = y - R < fy ? fy : y - R, y1 = y + R > fy + fh - 1 ? fy + fh - 1 : y + R;
                const int x0 = x - R < fx ? fx : x - R, x1 = x + R > fx + fw - 1 ? fx + fw - 1 : x + R;
                q = 0.0; s = 0.0;
                for (int yy = y0; yy <= y1; yy++) {
                    const size_t row = (size_t)(yy - fy) * fw - fx;
                    for (int xx = x0; xx <= x1; xx++) {
                        const int* g1 = G + (row + xx) * 3;
                        const double w = wtab[abs(g1[0] - g0[0]) + abs(g1[1] - g0[1]) + abs(g1[2] - g0[2])];
                        const double pv = (double)raw[row + xx];
                        q += pv * w;
                        s += fabs(pv) * w;
                    }
                }
            } else {
                q = (double)raw[ci];
                s = fabs(q);
            }
            if (with_check && !label_valid(plane, x, y, tw, th, c->min_disp, c->max_disp)) q = s = (double)COST_FOR_INVALID;
            out_q[o] = q;
            out_scale[o] = s;
        }
}

/* returns -1 for an unknown filter or a bilateral sig2 that is not positive */
int oracle_filter_unary_batch(void* p, int mode, int ncalls, const int* frects, const int* trects, const float* planes, double* out_q,
                              double* out_scale, int with_check, int filter, int windR, double sig2) {
    oracle_ctx* c = (oracle_ctx*)p;
    if (filter != ORACLE_FILTER_BILATERAL && filter != ORACLE_FILTER_NONE) return -1;
    if (filter == ORACLE_FILTER_BILATERAL && !(sig2 > 0)) return -1;
    double wtab[766];
    for (int s = 0; s < 766; s++) wtab[s] = exp(-(double)s / sig2);
#pragma omp parallel
    {
        filter_scratch sc = {0, NULL, NULL};
#pragma omp for schedule(dynamic, 1)
        for (int i = 0; i < ncalls; i++)
            oracle_filter_unary_s(c, mode, frects + 4 * i, trects + 4 * i, planes + 4 * i, out_q, out_scale, with_check, filter, windR,
                                  wtab, &sc);
        free(sc.raw); free(sc.guide);
    }
    return 0;
}

int oracle_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ------------------------------------------------------------------------------------------------------------------
 * Minimum cut of the expansion-move graph (FastGCStereo.h:424-557), for the graph-cut oracle (lexp_oracle.gc_step).
 * The graph is the one expansionMoveBK hands to the (un-vendored) Boykov-Kolmogorov library: nodes = pixels of a w x h
 * region; node s has the net terminal capacity tr[s] = (sum of its source weights) - (sum of its sink weights), i.e.
 * tr > 0: an arc source -> s, tr < 0: an arc s -> sink; cap[d][s] is the capacity of the arc s -> s + n_d for the four
 * forward neighbours d = 0 (+1,0), 1 (0,+1), 2 (-1,+1), 3 (+1,+1); the reverse arcs start at 0.
 * Result: mask[s] = 1 <=> BK's what_segment(s) == SOURCE <=> the sink is NOT reachable from s in the residual graph
 * of a maximum flow (oracle/maxflow/graph.h explains why that is BK's answer); *maxflow = value of the flow.
 * Algorithm: Dinic on the grid (BFS levels, iterative DFS), residuals in float as BK keeps them for
 * Graph<float, float, double>.
 * ------------------------------------------------------------------------------------------------------------------ */
static const int GDX[8] = {1, 0, -1, 1, -1, 0, 1, -1}, GDY[8] = {0, 1, 1, 1, 0, -1, -1, -1};   /* opposite of d: d ^ 4 */

int oracle_grid_mincut(int w, int h, const float* tr_in, const float* cap, unsigned char* mask, double* maxflow) {
    const int n = w * h;
    float* tr = (float*)malloc((size_t)n * sizeof(float));
    float* res = (float*)calloc((size_t)n * 8, sizeof(float));
    int* level = (int*)malloc((size_t)n * sizeof(int));
    int* it = (int*)malloc((size_t)n * sizeof(int));
    int* queue = (int*)malloc((size_t)n * sizeof(int));
    int* path = (int*)malloc((size_t)(n + 1) * sizeof(int));   /* direction taken at every node of the DFS path */
    int* pnode = (int*)malloc((size_t)(n + 1) * sizeof(int));
    if (!tr || !res || !level || !it || !queue || !path || !pnode) return -1;
    memcpy(tr, tr_in, (size_t)n * sizeof(float));
    for (int d = 0; d < 4; d++)
        for (int s = 0; s < n; s++) {
            const int x = s % w + GDX[d], y = s / w + GDY[d];
            if (x >= 0 && x < w && y >= 0 && y < h) res[(size_t)d * n + s] = cap[(size_t)d * n + s];
        }
    double flow = 0.0;
    for (;;) {
        int qh = 0, qt = 0, sink_seen = 0;
        for (int s = 0; s < n; s++) { level[s] = 0; if (tr[s] > 0) { level[s] = 1; queue[qt++] = s; } }
        while (qh < qt) {
            const int v = queue[qh++];
            if (tr[v] < 0) sink_seen = 1;
            for (int d = 0; d < 8; d++) {
                const int x = v % w + GDX[d], y = v / w + GDY[d];
                if (x < 0 || x >= w || y < 0 || y >= h) continue;
                const int u = y * w + x;
                if (res[(size_t)d * n + v] > 0 && !level[u]) { level[u] = level[v] + 1; queue[qt++] = u; }
            }
        }
        if (!sink_seen) break;
        for (int s = 0; s < n; s++) it[s] = 0;
        for (int s = 0; s < n; s++) {
            while (tr[s] > 0 && level[s] == 1) {
                int len = 0, v = s, found = 0;
                pnode[0] = s;
                for (;;) {
                    if (tr[v] < 0) { found = 1; break; }
                    int advanced = 0;
                    for (; it[v] < 8; it[v]++) {
                        const int d = it[v];
                        const int x = v % w + GDX[d], y = v / w + GDY[d];
                        if (x < 0 || x >= w || y < 0 || y >= h) continue;
                        const int u = y * w + x;
                        if (res[(size_t)d * n + v] > 0 && level[u] == level[v] + 1) { path[len++] = d; v = u; pnode[len] = v; advanced = 1; break; }
                    }
                    if (advanced) continue;
                    level[v] = -1;
                    if (len == 0) break;
                    len--; v = pnode[len];
                }
                if (!found) break;
                float f = tr[s];
                if (-tr[v] < f) f = -tr[v];
                for (int k = 0; k < len; k++) { const float r = res[(size_t)path[k] * n + pnode[k]]; if (r < f) f = r; }
                for (int k = 0; k < len; k++) { res[(size_t)path[k] * n + pnode[k]] -= f; res[(size_t)(path[k] ^ 4) * n + pnode[k + 1]] += f; }
                tr[s] -= f; tr[v] += f;
                flow += (double)f;
            }
        }
    }
    /* sink side: backward BFS from the nodes with sink capacity through arcs u -> v with residual capacity */
    int qh = 0, qt = 0;
    for (int s = 0; s < n; s++) { mask[s] = 1; if (tr[s] < 0) { mask[s] = 0; queue[qt++] = s; } }
    while (qh < qt) {
        const int v = queue[qh++];
        for (int d = 0; d < 8; d++) {   /* u = v + n_d reaches v through its arc of direction d ^ 4 */
            const int x = v % w + GDX[d], y = v / w + GDY[d];
            if (x < 0 || x >= w || y < 0 || y >= h) continue;
            const int u = y * w + x;
            if (mask[u] && res[(size_t)(d ^ 4) * n + u] > 0) { mask[u] = 0; queue[qt++] = u; }
        }
    }
    if (maxflow) *maxflow = flow;
    free(tr); free(res); free(level); free(it); free(queue); free(path); free(pnode);
    return 0;
}
