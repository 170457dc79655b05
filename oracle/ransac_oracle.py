"""CPU oracle of the device RansacProposer (csrc/lexp_ransac.cuh).  TEST INFRASTRUCTURE ONLY.

RansacProposer::getNextProposal -> RANSACPlane(coord, disps, 1.0) (Proposer.h:155-312) for one cell, restated under the
contract of DESIGN.md section 3f, which replaces the two parts of the reference that cannot be reproduced:
  * the random stream: sample s of a (cell, step) takes three draws from CvRng{pm_rng_state(seed, cell_id)},
    i0 = uniform_int(0, n), i1 = uniform_int(0, n - 1), i2 = uniform_int(0, n - 2), mapped to distinct indices (the first three
    entries of a uniform permutation; std::random_shuffle draws from the process-global rand()),
  * cv::solve(DECOMP_SVD): the minimum-norm least-squares solution in double on the uncentred (x, y, 1) rows, rounded once to
    float.  OpenCV drops singular values <= 2 DBL_EPSILON * sum (also in its float solve, see DESIGN.md section 3f): for integer
    coordinates that is the exact rank of the rows, which gram_rank computes in integers.  A full-rank system is solved in
    coordinates centred on the unit region (same solution, far better conditioned).  Route: the Gram matrix of the integer
    coordinates exactly, A^T b as a correctly rounded sum (math.fsum; double-double on the device), then a fixed sequence of IEEE
    double operations (cyclic Jacobi on the 3x3 Gram matrix, back-substitution over the kept eigenpairs) that the kernel performs
    operation for operation.
Everything else is the reference's control flow, including two details that decide the result:
  * the refit takes the inliers among the FIRST no_i points only (`for (i = 0, j = 0; i < no_i; i++) if (v(i))`, Proposer.h:207),
  * computeSampleCount converts with x86-64's rule: a quotient outside the int range (or NaN) becomes INT_MIN, then 1.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import lexp_oracle as O

MAX_SAM = 500                                   # RansacProposer(K, MAX_SAM = 500, conf = 0.95)
CONF = float(np.float32(0.95))                  # the float member widened to double at the call
LOG_1M_CONF = math.log(1.0 - CONF)              # = kRansacLog1mConf of the kernel
JACOBI_SWEEPS = 8
INT_MIN = -2147483648


def cvt_int_x86(r):
    """(int)r as x86-64's cvttsd2si computes it: truncation toward zero, INT_MIN when r is NaN or outside the int range."""
    if not (-2147483649.0 < r < 2147483648.0):
        return INT_MIN
    return int(r)


def compute_sample_count(ni, pt_num, pf=3, conf=CONF):
    """RansacProposer::computeSampleCount (Proposer.h:230-250)."""
    q = 1.0
    a, b = float(ni - pf + 1), float(pt_num - pf + 1)
    while a <= ni:
        q *= a / b
        a += 1.0
        b += 1.0
    if (1.0 - q) < 1e-4:
        cnt = 1
    else:
        lq = math.log(1.0 - q)
        num = LOG_1M_CONF if conf == CONF else math.log(1.0 - conf)
        cnt = cvt_int_x86(num / lq if lq != 0.0 else -math.inf)   # log(1) = +0: -inf as the IEEE division gives it
    return max(cnt, 1)


def draw_triple(rng: O.CvRNG, n):
    """Three draws -> three distinct row-major indices of the unit region (the first entries of a uniform permutation)."""
    i0 = rng.uniform_int(0, n)
    i1 = rng.uniform_int(0, n - 1)
    i2 = rng.uniform_int(0, n - 2)
    i1 += int(i1 >= i0)
    lo, hi = min(i0, i1), max(i0, i1)
    i2 += int(i2 >= lo)
    i2 += int(i2 >= hi)
    return i0, i1, i2


def gram_rank(G):
    """Rank of A = rows (x, y, 1), exactly, from the integer Gram matrix: 0 without points, 1 if all points coincide, 2 if they are
    collinear, else 3 (the determinant of the centred scatter matrix n^2 S = [[n Sxx - Sx^2, ..]] in exact integers)."""
    n = G[2][2]
    if n == 0:
        return 0
    sxx = n * G[0][0] - G[0][2] * G[0][2]
    syy = n * G[1][1] - G[1][2] * G[1][2]
    sxy = n * G[0][1] - G[0][2] * G[1][2]
    if sxx == 0 and syy == 0:
        return 1
    return 2 if sxx * syy == sxy * sxy else 3


def minnorm_solve(G, g, rank, rounded=True):
    """The contract's cv::solve(DECOMP_SVD): G = A^T A (exact integers, 3x3), g = A^T b (3 doubles).  Cyclic Jacobi on G, then
    N = sum over the kept eigenpairs of v_i (v_i . g) / lambda_i; the 3 - rank smallest eigenvalues are dropped, the rank exact.
    Python floats are IEEE doubles without contraction: this is the kernel's operation sequence (ransac_minnorm).  Returns
    float32[3], or the three doubles when not `rounded`."""
    a = [[float(G[i][j]) for j in range(3)] for i in range(3)]
    V = [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]
    for _ in range(JACOBI_SWEEPS):
        for p, q in ((0, 1), (0, 2), (1, 2)):
            apq = a[p][q]
            if apq == 0.0:
                continue
            tau = (a[q][q] - a[p][p]) / (2.0 * apq)
            t = 1.0 / (abs(tau) + math.sqrt(1.0 + tau * tau))
            if tau < 0.0:
                t = -t
            c = 1.0 / math.sqrt(1.0 + t * t)
            s = t * c
            a[p][p] = a[p][p] - t * apq
            a[q][q] = a[q][q] + t * apq
            a[p][q] = a[q][p] = 0.0
            r = 3 - p - q
            arp, arq = a[r][p], a[r][q]
            a[r][p] = a[p][r] = c * arp - s * arq
            a[r][q] = a[q][r] = s * arp + c * arq
            for k in range(3):
                vkp, vkq = V[k][p], V[k][q]
                V[k][p] = c * vkp - s * vkq
                V[k][q] = s * vkp + c * vkq
    lam = [a[0][0], a[1][1], a[2][2]]
    keep = [True, True, True]
    for _ in range(3 - rank):   # drop the smallest eigenvalues (the first of equal ones)
        i = min((j for j in range(3) if keep[j]), key=lambda j: lam[j])
        keep[i] = False
    N = [0.0, 0.0, 0.0]
    for i in range(3):
        if keep[i]:
            d = (V[0][i] * g[0] + V[1][i] * g[1]) + V[2][i] * g[2]
            w = d / lam[i]
            for k in range(3):
                N[k] = N[k] + V[k][i] * w
    return np.array(N, dtype=np.float32) if rounded else N


def fit_plane(xs, ys, b, centre=(0, 0)):
    """The contract's solve on the rows (x, y, 1) / right-hand side b (float32) of the given points.  Full rank: solved in coordinates
    centred on the integer point `centre` (the unit region's centre), c = c' - (a cx + b cy); rank < 3: the minimum-norm solution of
    the uncentred rows."""
    b = np.asarray(b, np.float32)
    if not np.isfinite(b).all():
        return np.full(3, np.nan, np.float32)      # never an inlier of anything (IEEE): the kernel's value may differ, its count cannot
    xs = np.asarray(xs, np.int64)
    ys = np.asarray(ys, np.int64)
    cx, cy = int(centre[0]), int(centre[1])
    bd = b.astype(np.float64)

    def gram(X, Y):
        sx, sy = int(X.sum()), int(Y.sum())
        G = [[int((X * X).sum()), int((X * Y).sum()), sx], [int((X * Y).sum()), int((Y * Y).sum()), sy], [sx, sy, len(X)]]
        g = [math.fsum((X.astype(np.float64) * bd).tolist()), math.fsum((Y.astype(np.float64) * bd).tolist()), math.fsum(bd.tolist())]
        return G, g
    G, g = gram(xs, ys)
    rank = gram_rank(G)
    if rank < 3:
        return minnorm_solve(G, g, rank)
    Gc, gc = gram(xs - cx, ys - cy)
    N = minnorm_solve(Gc, gc, 3, rounded=False)
    N[2] = N[2] - (N[0] * float(cx) + N[1] * float(cy))
    return np.array(N, dtype=np.float32)


def unit_snapshot(cur_label, unit):
    """RansacProposer::startIterations: row-major (x, y) of the unit region and disps = (v0 x + v1 y) + v2 in float."""
    ux, uy, uw, uh = (int(v) for v in unit)
    Y, X = np.mgrid[uy:uy + uh, ux:ux + uw]
    lab = np.asarray(cur_label[uy:uy + uh, ux:ux + uw], np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        d = (lab[..., 0] * X.astype(np.float32) + lab[..., 1] * Y.astype(np.float32)) + lab[..., 2]
    return X.ravel().astype(np.int64), Y.ravel().astype(np.int64), d.ravel().astype(np.float32)


def inliers(N, X, Y, disp):
    """dist = |(float)(((double)x a + (double)y b) + c) - disp| < 1.0f (the float gemm of OpenCV accumulates in double)."""
    a, b, c = (float(v) for v in np.asarray(N, np.float32))
    with np.errstate(invalid="ignore", over="ignore"):
        pred = ((X.astype(np.float64) * a + Y.astype(np.float64) * b) + c).astype(np.float32)
        return np.abs(pred - disp) < np.float32(1.0)


def ransac_points(X, Y, disp, state, centre, max_sam=MAX_SAM, fit=None):
    """RANSACPlane on explicit points (`fit`: another solve, for measurements).  Returns (plane float32[4], trace) with one trace entry per sample:
    (triple, no_i, refit, no (-1 without refit), accepted, max_sam after the sample)."""
    n = len(X)
    trace = []
    if n <= 3:                                   # no sample can have more than 3 inliers
        return np.zeros(4, np.float32), trace
    rng = O.CvRNG(state)
    max_i, no_sam, no_i_c = 3, 0, 0
    result = np.zeros(3, np.float32)
    while no_sam < max_sam:
        no_sam += 1
        tri = draw_triple(rng, n)
        idx = np.array(tri)
        N = (fit or fit_plane)(X[idx], Y[idx], disp[idx], centre)
        v = inliers(N, X, Y, disp)
        no_i = int(v.sum())
        refit, no, acc = False, -1, False
        if max_i < no_i:
            refit = True
            sel = np.nonzero(v[:no_i])[0]       # Proposer.h:207: i < no_i
            Nr = (fit or fit_plane)(X[sel], Y[sel], disp[sel], centre)
            no = int(inliers(Nr, X, Y, disp).sum())
            if no > no_i_c:
                acc = True
                result, no_i_c, max_i = Nr, no, no_i
                max_sam = min(max_sam, compute_sample_count(no, n))
        trace.append((tri, no_i, refit, no, acc, max_sam))
    return np.array([result[0], result[1], result[2], 0.0], np.float32), trace


def ransac_proposal(state, cur_label, unit, max_sam=MAX_SAM, fit=None):
    """RansacProposer(1): startIterations on cur_label, then getNextProposal, with the random stream `state`
    (= oracle.lexp_oracle.pm_rng_state(seed, cell_id)).  Returns (plane, trace)."""
    X, Y, d = unit_snapshot(cur_label, unit)
    ux, uy, uw, uh = (int(v) for v in unit)
    return ransac_points(X, Y, d, state, (ux + uw // 2, uy + uh // 2), max_sam, fit)

