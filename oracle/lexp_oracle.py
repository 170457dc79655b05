"""CPU oracle for the LocalExpStereo unary-cost hot path.  TEST INFRASTRUCTURE ONLY.

This module restates, in numpy, the arithmetic of the reference's hot path
(`/root/reference/LocalExpansionStereo/*`; citations below are file:line in that
directory).  It is the *checker* for the CUDA path: only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s `cpu_baseline` / `--impl reference`
legs may import it.  Nothing under `localexpstereo_b200/` imports it.

PARITY STATUS: **pinned by the reference's own code.**  The reference ships no
tests, golden vectors or known-answer values for this path (SURVEY.md section 4
and 8c), and its own build (Visual Studio + NuGet OpenCV 3.1) cannot run here; but
the classes on the path -- CostVolumeEnergy, NaiveStereoEnergy,
FastGuidedImageFilter<double>, LayerManager, RandomProposer -- compile with g++
from the headers where they lie (`oracle/build_ref.py` -> `oracle/_ref/`, over the
small cv:: layer of `oracle/cvshim/`).  What pins this restatement:
  * `tests/test_ref_pin.py`: costs (every cell class, both views, with and
    without the validity check, NaN / out-of-range / steep planes, MIN != 0),
    validity masks, guided-filter statistics, cell geometry, Plane helpers and
    cv::RNG-driven labels are compared with the compiled reference: costs agree
    bit for bit on synthetic scenes and to 1 float ulp on a natural image,
  * the cv:: layer's primitives (box filter, warpAffine, getAffineTransform,
    cvtColor, Sobel) and this file's own (`tests/test_oracle.py`) are checked
    against the real OpenCV kernels (`cv2` 4.13 wheel, the only OpenCV in the image),
  * `tests/golden/*.npz` are OUTPUTS OF THE COMPILED REFERENCE
    (`tests/golden/make_golden.py`); they travel to the GPU box, which has no
    /root/reference,
  * `oracle/lexp_oracle.c` is an independent plain-C restatement held to both.
Residual freedom: the cv:: layer is this repository's reading of OpenCV 3.1's
documented behaviour (checked on 4.13), not OpenCV 3.1 itself.

Conventions: rect = (x, y, w, h) in image coordinates (cv::Rect); plane =
(a, b, c, v) float32 (Plane.h:4-8); volume = float32[D][H][W] (main.cpp:353-354);
guide image = uint8[H][W][3] in OpenCV BGR channel order.
"""
from __future__ import annotations

import numpy as np

COST_FOR_INVALID = np.float32(1000000.0)  # StereoEnergy.h:45

f32 = np.float32


# ----------------------------------------------------------------------------
# Plane (Plane.h:4-106)
# ----------------------------------------------------------------------------
def create_plane(nx, ny, nz, z, x, y, v=0.0):
    """Plane::CreatePlane (Plane.h:14-32): all arithmetic in float."""
    nx, ny, nz, z, x, y = (f32(t) for t in (nx, ny, nz, z, x, y))
    a = f32(-nx / nz)
    b = f32(-ny / nz)
    c = f32(f32(z - f32(a * x)) - f32(b * y))
    return np.array([a, b, c, f32(v)], dtype=np.float32)


def plane_normal(plane):
    """Plane::GetNormal (Plane.h:42-50): sqrt in double, then cast to float."""
    a, b = f32(plane[0]), f32(plane[1])
    # `1.0 + a*a + b*b`: a*a is float*float (rounded to float), then promoted to double
    nz = f32(1.0 / np.sqrt(1.0 + float(f32(a * a)) + float(f32(b * b))))
    nx = f32(-a * nz)
    ny = f32(-b * nz)
    return np.array([nx, ny, nz], dtype=np.float32)


def plane_get_z(plane, x, y):
    """Plane::GetZ (Plane.h:51-58): (a*x + b*y) + c in float, no contraction."""
    a, b, c = f32(plane[0]), f32(plane[1]), f32(plane[2])
    x = np.asarray(x, dtype=np.float32)
    y = np.asarray(y, dtype=np.float32)
    return (a * x + b * y) + c


# ----------------------------------------------------------------------------
# cv::RNG restatement (OpenCV core, multiply-with-carry; used by
# StereoEnergy.h:120-129, Proposer.h:38-45,120-148, Utilities.hpp:254-261)
# ----------------------------------------------------------------------------
class CvRNG:
    """cv::RNG: state = (uint32)state * 4164903690 + (state >> 32)."""

    def __init__(self, seed=0xFFFFFFFF):
        self.state = int(seed) & 0xFFFFFFFFFFFFFFFF
        if self.state == 0:
            self.state = 0xFFFFFFFF

    def next(self):
        self.state = ((self.state & 0xFFFFFFFF) * 4164903690 + (self.state >> 32)) & 0xFFFFFFFFFFFFFFFF
        return self.state & 0xFFFFFFFF

    def uniform_int(self, a, b):
        return a if a == b else int(self.next() % (b - a) + a)

    def uniform_float(self, a, b):
        a, b = f32(a), f32(b)
        r = f32(f32(self.next()) * f32(2.3283064365386962890625e-10))
        return f32(f32(r * f32(b - a)) + a)

    def uniform_double(self, a, b):
        t = self.next()
        t = (t << 32) | self.next()
        # (uint64)t * 5.4210108624275221700372640043497e-20  -> [0, 1)
        r = float(t) * 5.4210108624275221700372640043497e-20
        return r * (b - a) + a


def random_unit_vector(rng: CvRNG, theta_range=np.pi):
    """cvutils::getRandomUnitVector (Utilities.hpp:254-261)."""
    theta = rng.uniform_double(0.0, theta_range)
    phi = rng.uniform_double(0.0, np.pi * 2.0)
    ct, st = np.cos(theta), np.sin(theta)
    cp, sp = np.cos(phi), np.sin(phi)
    return np.array([st * cp, st * sp, ct], dtype=np.float64)


def create_random_label(rng: CvRNG, sx, sy, min_disp, max_disp):
    """StereoEnergy::createRandomLabel (StereoEnergy.h:120-129), MAX_VDISPARITY == 0."""
    zs = rng.uniform_float(min_disp, max_disp)
    n = random_unit_vector(rng, np.pi / 3)
    nf = n.astype(np.float32)  # Vec3d -> Vec<float,3> conversion at the call
    return create_plane(nf[0], nf[1], nf[2], zs, f32(sx), f32(sy), 0.0)


def random_proposal(rng: CvRNG, plane_in, sx, sy, m, min_disp, max_disp):
    """RandomProposer::getNextProposal (Proposer.h:120-148) for a given source
    label `plane_in` taken at pixel (sx, sy); m = outerIter + iter; MAX_VDISPARITY == 0."""
    zs = plane_get_z(plane_in, f32(sx), f32(sy))
    dz = f32(f32(max_disp - min_disp) * f32(np.power(f32(0.5), m + 1)))
    minz = max(f32(min_disp), f32(zs - dz))
    maxz = min(f32(max_disp), f32(zs + dz))
    zs = rng.uniform_float(minz, maxz)
    nr = f32(f32(1.0) * f32(np.power(f32(0.5), m)))
    rv = random_unit_vector(rng).astype(np.float32)
    nv = plane_normal(plane_in) + rv * nr
    nv = nv.astype(np.float32)
    nrm = np.sqrt(float(nv[0]) * float(nv[0]) + float(nv[1]) * float(nv[1]) + float(nv[2]) * float(nv[2]))
    nv = (nv.astype(np.float64) * (1.0 / nrm)).astype(np.float32)   # cv::Vec / double = Vec * (1. / alpha)  (matx.hpp)
    return create_plane(nv[0], nv[1], nv[2], zs, f32(sx), f32(sy), plane_in[3])


# ----------------------------------------------------------------------------
# LayerManager::addLayer (LayerManager.h:88-185)
# ----------------------------------------------------------------------------
def _clip(r, W, H):
    x0, y0 = max(r[0], 0), max(r[1], 0)
    x1, y1 = min(r[0] + r[2], W), min(r[1] + r[3], H)
    if x1 <= x0 or y1 <= y0:
        return (0, 0, 0, 0)  # cv::Rect & of disjoint rects is the empty Rect()
    return (x0, y0, x1 - x0, y1 - y0)


def make_layer(W, H, windR, u):
    """Returns dict(heightBlocks, widthBlocks, unit, shared, filter, groups)."""
    minsize = max(2, u // 2)
    frac_h, frac_w = H % u, W % u
    split_h = 1 if frac_h >= minsize else 0
    split_w = 1 if frac_w >= minsize else 0
    hb, wb = H // u + split_h, W // u + split_w
    unit, shared, filt = [], [], []
    for i in range(hb):
        for j in range(wb):
            unit.append(_clip((j * u, i * u, u, u), W, H))
            shared.append(_clip(((j - 1) * u, (i - 1) * u, 3 * u, 3 * u), W, H))
            filt.append(_clip(((j - 1) * u - windR, (i - 1) * u - windR, 3 * u + 2 * windR, 3 * u + 2 * windR), W, H))
    if split_w == 0:
        for i in range(hb):
            x1 = i * wb + wb - 1
            r = unit[x1]
            unit[x1] = (r[0], r[1], r[2] + frac_w, r[3])
        if wb >= 2:
            for i in range(hb):
                x1 = i * wb + wb - 2
                r = shared[x1]
                shared[x1] = (r[0], r[1], r[2] + frac_w, r[3])
                r = filt[x1]
                filt[x1] = _clip((r[0], r[1], r[2] + frac_w, r[3]), W, H)
    if split_h == 0:
        for j in range(wb):
            y1 = (hb - 1) * wb + j
            r = unit[y1]
            unit[y1] = (r[0], r[1], r[2], r[3] + frac_h)
        if hb >= 2:
            for j in range(wb):
                y1 = (hb - 2) * wb + j
                r = shared[y1]
                shared[y1] = (r[0], r[1], r[2], r[3] + frac_h)
                r = filt[y1]
                filt[y1] = _clip((r[0], r[1], r[2], r[3] + frac_h), W, H)
    groups = [[] for _ in range(16)]
    for i in range(hb):
        for j in range(wb):
            groups[(i % 4) * 4 + (j % 4)].append(i * wb + j)
    groups = [g for g in groups if g]
    return dict(heightBlocks=hb, widthBlocks=wb, unitSize=u, unit=unit, shared=shared, filter=filt, groups=groups)


# ----------------------------------------------------------------------------
# Box filter: cv::boxFilter(ksize=2R+1, normalize=false, BORDER_CONSTANT)
# (GuidedFilter.h:40-45).  OpenCV accumulates 32F/64F sources in double.
# ----------------------------------------------------------------------------
def box_sum(X, R):
    X64 = np.asarray(X, dtype=np.float64)
    h, w = X64.shape
    P = np.zeros((h + 2 * R + 1, w + 2 * R + 1), dtype=np.float64)
    P[R + 1:R + 1 + h, R + 1:R + 1 + w] = X64
    # windowed sums by explicit sliding accumulation along each axis (same
    # operation order as a running row/column sum; no integral-image cancellation)
    k = 2 * R + 1
    rows = np.zeros((h + 2 * R + 1, w), dtype=np.float64)
    acc = P[:, 1:k + 1].sum(axis=1)
    rows[:, 0] = acc
    for x in range(1, w):
        acc = acc + P[:, x + k] - P[:, x]
        rows[:, x] = acc
    out = np.zeros((h, w), dtype=np.float64)
    acc = rows[1:k + 1, :].sum(axis=0)
    out[0, :] = acc
    for y in range(1, h):
        acc = acc + rows[y + k, :] - rows[y, :]
        out[y, :] = acc
    return out.astype(np.asarray(X).dtype if np.asarray(X).dtype in (np.float32, np.float64) else np.float64)


def box_sum_fast(X, R):
    """Same quantity through a float64 summed-area table (used for big inputs;
    agrees with box_sum to ~1e-13 relative)."""
    X64 = np.asarray(X, dtype=np.float64)
    h, w = X64.shape
    S = np.zeros((h + 1, w + 1), dtype=np.float64)
    np.cumsum(X64, axis=0, out=S[1:, 1:])
    np.cumsum(S[1:, 1:], axis=1, out=S[1:, 1:])
    y0 = np.clip(np.arange(h) - R, 0, h)
    y1 = np.clip(np.arange(h) + R + 1, 0, h)
    x0 = np.clip(np.arange(w) - R, 0, w)
    x1 = np.clip(np.arange(w) + R + 1, 0, w)
    out = S[np.ix_(y1, x1)] - S[np.ix_(y0, x1)] - S[np.ix_(y1, x0)] + S[np.ix_(y0, x0)]
    dt = np.asarray(X).dtype
    return out.astype(dt if dt in (np.float32, np.float64) else np.float64)


# ----------------------------------------------------------------------------
# GuidedImageFilter<T> statistics (GuidedFilter.h:58-102) and
# FastGuidedImageFilter<T>::createSubregionFilter (:301-326)
# ----------------------------------------------------------------------------
class GuidedFilterStats:
    """One-time per-image statistics: realI, mean_I_{r,g,b}, inv{rr,rg,rb,gg,gb,bb}."""

    def __init__(self, I8, R, eps, dtype=np.float64, scaling=1.0 / 255, box=box_sum_fast):
        T = np.dtype(dtype).type
        self.T, self.R, self.eps, self.box = T, int(R), float(eps), box
        I8 = np.asarray(I8)
        assert I8.ndim == 3 and I8.shape[2] == 3
        if T is np.float64:
            real = I8.astype(np.float64) * float(scaling)  # convertTo(..., DEPTH, scaling) (:62-65)
        else:
            real = I8.astype(np.float32) * np.float32(scaling)
        self.I = [np.ascontiguousarray(real[:, :, k]) for k in range(3)]  # cv::split (:67)
        ones = np.ones(real.shape[:2], dtype=T)
        bx = lambda X: box(X.astype(T), self.R)
        N = bx(ones)  # (:69)
        self.N_image = N
        Ir, Ig, Ib = self.I
        self.mean = [bx(Ir) / N, bx(Ig) / N, bx(Ib) / N]  # (:70-72)
        mr, mg, mb = self.mean
        e = T(eps)
        vrr = bx(Ir * Ir) / N - mr * mr + e  # (:79-84)
        vrg = bx(Ir * Ig) / N - mr * mg
        vrb = bx(Ir * Ib) / N - mr * mb
        vgg = bx(Ig * Ig) / N - mg * mg + e
        vgb = bx(Ig * Ib) / N - mg * mb
        vbb = bx(Ib * Ib) / N - mb * mb + e
        irr = vgg * vbb - vgb * vgb  # (:87-92)
        irg = vgb * vrb - vrg * vbb
        irb = vrg * vgb - vgg * vrb
        igg = vrr * vbb - vrb * vrb
        igb = vrb * vrg - vrr * vgb
        ibb = vrr * vgg - vrg * vrg
        det = irr * vrr + irg * vrg + irb * vrb  # (:94)
        self.inv = [irr / det, irg / det, irb / det, igg / det, igb / det, ibb / det]  # (:96-101)

    def stats_f32(self):
        """[9][H][W] float32: mean_r, mean_g, mean_b, irr, irg, irb, igg, igb, ibb."""
        return np.stack([m.astype(np.float32) for m in self.mean] + [m.astype(np.float32) for m in self.inv])


def subregion_N(rect, R, T=np.float64):
    """N = boxfilter(ones(rect.size())) (GuidedFilter.h:324): window counts
    clipped at the *filterRect* border."""
    _, _, w, h = rect
    xs = np.arange(w)
    ys = np.arange(h)
    nx = np.minimum(xs + R, w - 1) - np.maximum(xs - R, 0) + 1
    ny = np.minimum(ys + R, h - 1) - np.maximum(ys - R, 0) + 1
    return (ny[:, None] * nx[None, :]).astype(T)


def guided_filter_sub(stats: GuidedFilterStats, rect, p_f32):
    """GuidedImageFilter<T>::filter -> filter_raw (GuidedFilter.h:248-266, 142-247)
    on the sub-region filter created for `rect` (:301-326).  Returns float32."""
    T, R, box = stats.T, stats.R, stats.box
    x, y, w, h = rect
    sl = (slice(y, y + h), slice(x, x + w))
    I = [c[sl] for c in stats.I]
    m = [c[sl] for c in stats.mean]
    irr, irg, irb, igg, igb, ibb = [c[sl] for c in stats.inv]
    N = subregion_N(rect, R, T)
    p = p_f32.astype(T)  # (:250-252)
    bx = lambda X: box(np.ascontiguousarray(X, dtype=T), R)
    Bp = bx(p)  # (:145)
    Br, Bg, Bb_ = bx(I[0] * p), bx(I[1] * p), bx(I[2] * p)  # (:151-172)
    mp = Bp / N  # (:206)
    cr = Br / N - m[0] * mp  # (:212-214)
    cg = Bg / N - m[1] * mp
    cb = Bb_ / N - m[2] * mp
    ar = irr * cr + irg * cg + irb * cb  # (:216-218)
    ag = irg * cr + igg * cg + igb * cb
    ab = irb * cr + igb * cg + ibb * cb
    bb = mp - ar * m[0] - ag * m[1] - ab * m[2]  # (:220)
    q = (bx(bb) + bx(ar) * I[0] + bx(ag) * I[1] + bx(ab) * I[2]) / N  # (:224-227, :243)
    return q.astype(np.float32)  # (:260-263)


# ----------------------------------------------------------------------------
# CostVolumeEnergy (CostVolumeEnergy.h:55-183) and validity (StereoEnergy.h:560-610)
# ----------------------------------------------------------------------------
def sample_plane_cost(vol, rect, plane, th_col, min_disp=0.0, max_disp=None):
    """HOT LOOP 1 (CostVolumeEnergy.h:69-98), interpolate == 1.  Returns pIL float32[h][w]."""
    D = vol.shape[0]
    MIN = f32(min_disp)
    MAX = f32(D - 1 if max_disp is None else max_disp)
    D0 = int(-float(MIN))
    x, y, w, h = rect
    a, b, c = f32(plane[0]), f32(plane[1]), f32(plane[2])
    ys = np.arange(y, y + h, dtype=np.int64)
    xs = np.arange(x, x + w, dtype=np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        d_base = (b * ys.astype(np.float32) + c).astype(np.float32)  # (:73)
        d = (a * xs.astype(np.float32))[None, :] + d_base[:, None]  # (:76)
        d = d.astype(np.float32)
        lo = d < MIN
        hi = (~lo) & (d >= MAX)
        bad = (~lo) & (~hi) & ~np.isfinite(d)
        ok = ~(lo | hi | bad)
        dd = np.where(ok, d, f32(0))
        d0 = dd.astype(np.int32) + D0  # int(d): truncation toward zero (:83)
        f1 = (dd - np.floor(dd)).astype(np.float32)  # (:85)
        f0 = (f32(1.0) - f1).astype(np.float32)
        d1 = d0 + 1
        oob = ok & ((d1 >= D) | (d0 < 0))  # (:87-90)
        d0c = np.clip(d0, 0, D - 1)
        d1c = np.clip(d1, 0, D - 1)
        Y = ys[:, None] + np.zeros((1, w), dtype=np.int64)
        X = xs[None, :] + np.zeros((h, 1), dtype=np.int64)
        v0 = vol[d0c, Y, X]
        v1 = vol[d1c, Y, X]
        C = (f0 * v0).astype(np.float32) + (f1 * v1).astype(np.float32)  # (:92)
        C = np.where(lo, vol[0][Y, X], C)  # (:78)
        C = np.where(hi, vol[D - 1][Y, X], C)  # (:79)
        C = np.where(bad | oob, COST_FOR_INVALID, C).astype(np.float32)  # (:80,:89)
        th = f32(th_col)
        p = np.where(th < C, th, C).astype(np.float32)  # std::min(C, th_col) (:96)
    return p


def is_valid_label(plane, rect, min_disp, max_disp):
    """StereoEnergy::IsValiLabel(Plane, Rect) (StereoEnergy.h:577-610) -> bool[h][w].
    ds follows cvutils::channelSum(coordinates(pos).mul(label.toScalar()))
    (Utilities.hpp:224-229): float products summed left to right,
    ((x*a + y*b) + 1*c) + 0*v  (order verified against cv2.reduce, see tests)."""
    x, y, w, h = rect
    a, b, c, v = (f32(t) for t in plane[:4])
    MIN, MAX = f32(min_disp), f32(max_disp)
    with np.errstate(invalid="ignore", over="ignore"):
        a5 = f32(a * f32(5))
        b5 = f32(b * f32(5))
        if w == 1 and h == 1:  # 1x1 fast path (:579-583 -> :560-574): Plane::GetZ(cv::Point)
            ds = np.array([[(a * f32(x) + b * f32(y)) + c]], dtype=np.float32)
        else:
            xs = np.arange(x, x + w).astype(np.float32)[None, :]
            ys = np.arange(y, y + h).astype(np.float32)[:, None]
            ds = ((xs * a + ys * b).astype(np.float32) + c * f32(1)).astype(np.float32) + f32(0) * v
            ds = ds.astype(np.float32)
        ok = (ds >= MIN) & (ds <= MAX)
        for sa, sb in ((1, 1), (1, -1), (-1, 1), (-1, -1)):
            t = (ds + a5) if sa > 0 else (ds - a5)
            t = t.astype(np.float32)
            t = (t + b5) if sb > 0 else (t - b5)
            t = t.astype(np.float32)
            ok &= (t >= MIN) & (t <= MAX)
    return ok


class CostVolumeEnergyOracle:
    """CostVolumeEnergy (CostVolumeEnergy.h:6-184) with filterName "GF" (T=double,
    default, main.cpp:73) or "GFfloat" (T=float) or "" (no filter)."""

    def __init__(self, imL, imR, volL, volR, windR, eps, th_col, max_disp, min_disp=0.0,
                 filter_name="GF", box=box_sum_fast):
        self.im = [np.asarray(imL), np.asarray(imR) if imR is not None else None]
        self.vol = [volL, volR]
        self.windR, self.eps, self.th_col = int(windR), float(eps), f32(th_col)
        self.MAX, self.MIN = f32(max_disp), f32(min_disp)
        self.filter_name = filter_name
        self.filter = [None, None]
        if filter_name in ("GF", "GFfloat"):
            T = np.float64 if filter_name == "GF" else np.float32
            for m in range(2):
                if self.im[m] is not None:
                    self.filter[m] = GuidedFilterStats(self.im[m], self.windR // 2, eps, T, box=box)  # (:30-31)

    def raw(self, filter_rect, plane, mode=0):
        return sample_plane_cost(self.vol[mode], filter_rect, plane, self.th_col, self.MIN, self.MAX)

    def compute_unary_potential_without_check(self, filter_rect, target_rect, plane, mode=0):
        """Returns float32[th][tw]: the values written to costs(targetRect - filterRect.tl()) (:169-171)."""
        p = self.raw(filter_rect, plane, mode)
        fx, fy, _, _ = filter_rect
        tx, ty, tw, th = target_rect
        q = guided_filter_sub(self.filter[mode], filter_rect, p) if self.filter_name else p
        return q[ty - fy:ty - fy + th, tx - fx:tx - fx + tw].copy()

    def compute_unary_potential(self, filter_rect, target_rect, plane, mode=0):
        out = self.compute_unary_potential_without_check(filter_rect, target_rect, plane, mode)
        valid = is_valid_label(plane, target_rect, self.MIN, self.MAX)  # (:179)
        out[~valid] = COST_FOR_INVALID  # (:180-182)
        return out


# ----------------------------------------------------------------------------
# Volume preparation (main.cpp:146-199)
# ----------------------------------------------------------------------------
def fill_out_of_view(vol, mode, margin=0):
    """fillOutOfView (main.cpp:146-176), in place."""
    D, H, W = vol.shape
    for d in range(D):
        k = d + margin
        if mode == 0:
            if k > 0:
                vol[d, :, :k] = vol[d, :, k:k + 1]
        else:
            if k > 0:
                vol[d, :, W - k:] = vol[d, :, W - k - 1:W - k]
    return vol


def convert_volume_l2r(vol, margin=0):
    """convertVolumeL2R (main.cpp:178-199)."""
    D, H, W = vol.shape
    dst = vol.copy()
    for d in range(D):
        dst[d, :, :W - d] = vol[d, :, d:]
        edge1 = vol[d, :, W - 1 - margin].copy()
        edge0 = vol[d, :, d + margin].copy()
        for x in range(W - 1 - d - margin, W):
            dst[d, :, x] = edge1
        for x in range(margin):
            dst[d, :, x] = edge0
    return dst


# ----------------------------------------------------------------------------
# Synthetic inputs (SURVEY.md section 8d) -- shared by tests and bench so that the
# GPU arm, the oracle and the CPU baseline see identical data.
# ----------------------------------------------------------------------------
def synthetic_image(H, W, seed):
    """8UC3 guide: smooth random field stretched to 0..255 plus +-8 white noise."""
    rng = np.random.default_rng(seed)
    img = np.empty((H, W, 3), dtype=np.uint8)
    # separable binomial-ish blur (sigma ~ 3) of uniform noise, numpy only
    k = np.exp(-0.5 * (np.arange(-9, 10) / 3.0) ** 2)
    k /= k.sum()
    for c in range(3):
        z = rng.random((H + 18, W + 18))
        zz = np.zeros((H + 18, W))
        for i, kk in enumerate(k):  # separable 19-tap blur as shifted adds
            zz += kk * z[:, i:i + W]
        z = np.zeros((H, W))
        for i, kk in enumerate(k):
            z += kk * zz[i:i + H, :]
        z = (z - z.min()) / max(z.max() - z.min(), 1e-12) * 255.0
        z = z + rng.integers(-8, 9, size=(H, W))
        img[:, :, c] = np.clip(np.rint(z), 0, 255).astype(np.uint8)
    return img


def synthetic_volume(D, H, W, seed):
    rng = np.random.default_rng(seed)
    return rng.random((D, H, W), dtype=np.float32)


def synthetic_planes(cells_unit, n_steps, D, seed):
    """Per cell, per step: createRandomLabel anchored at a random pixel of the unit
    cell for step 0, RandomProposer perturbations (m = step-1) of it afterwards."""
    rng = CvRNG(seed if seed else 1)
    out = np.zeros((n_steps, len(cells_unit), 4), dtype=np.float32)
    for i, (ux, uy, uw, uh) in enumerate(cells_unit):
        n = rng.uniform_int(0, uw * uh)
        sx, sy = ux + n % uw, uy + n // uw
        base = create_random_label(rng, sx, sy, 0.0, float(D - 1))
        out[0, i] = base
        for s in range(1, n_steps):
            out[s, i] = random_proposal(rng, base, sx, sy, s - 1, 0.0, float(D - 1))
    return out


# ----------------------------------------------------------------------------
# NaiveStereoEnergy (StereoEnergy.h:629-764): image-based unary term of `-mode MiddV2`
# (BASELINE.json configs[0]).  OpenCV calls restated: cvtColor(BGR2GRAY) on 32F, Sobel(ksize=1,
# scale=0.5, BORDER_REPLICATE), getAffineTransform, warpAffine(INTER_LINEAR, BORDER_REPLICATE)
# with its fixed-point coordinates (imgwarp.cpp: AB_BITS = 10, INTER_BITS = 5).
# ----------------------------------------------------------------------------
def build_exI(im8, alpha):
    """ExI = merge(I*(1-alpha), alpha*Sobel_x(gray)) as float32[H][W][4]  (StereoEnergy.h:647-662)."""
    I = np.asarray(im8).astype(np.float32)  # imL.convertTo(I[0], CV_32FC3) (StereoEnergy.h:96)
    # cv::cvtColor(BGR2GRAY) on CV_32F: B*0.114f + G*0.587f + R*0.299f in float, left to right (OpenCV 3.1 scalar path)
    gray = ((I[:, :, 0] * f32(0.114) + I[:, :, 1] * f32(0.587)).astype(np.float32) + I[:, :, 2] * f32(0.299)).astype(np.float32)
    gp = np.pad(gray, ((0, 0), (1, 1)), mode="edge")
    gx = ((gp[:, 2:] - gp[:, :-2]) * f32(0.5)).astype(np.float32)  # Sobel dx=1, ksize=1, scale 0.5, BORDER_REPLICATE (:654)
    s_col = f32(1.0 - float(f32(alpha)))  # `I[m] * (1.0 - params.alpha)`: double scale, applied in float by cvtScale
    ex = np.empty(I.shape[:2] + (4,), np.float32)
    ex[:, :, :3] = (I * s_col).astype(np.float32)
    ex[:, :, 3] = (gx * f32(alpha)).astype(np.float32)
    return ex


def _cv_round(x):
    """saturate_cast<int>(double) = cvRound: round half to even."""
    return np.rint(np.asarray(x, dtype=np.float64)).astype(np.int64)


def affine_inverse_for_plane(filter_rect, plane, mode):
    """The 2x3 double matrix cv::warpAffine uses (dst pixel -> source pixel) for the three float corner
    correspondences of StereoEnergy.h:704-727, computed the way the reference does: cv::getAffineTransform (6x6 system,
    Gaussian elimination with partial pivoting in double -- cv::solve DECOMP_LU) followed by the inversion at the top of
    cv::warpAffine.  Python floats are IEEE doubles and every operation below is a single rounded one, in the order of
    oracle/cvshim (the cv:: layer oracle/_ref is compiled over), so the matrix -- and with it every 1/32-pixel source
    coordinate -- is bit-identical to the compiled reference's; the CUDA path repeats the same sequence."""
    x, y, w, h = filter_rect
    sign = f32(-1.0) if mode else f32(1.0)
    x00, y00 = f32(x), f32(y)
    x11, y11 = f32(x00 + f32(w)), f32(y00 + f32(h))
    gz = lambda xx, yy: plane_get_z(plane, xx, yy)
    sx = [f32(x00 - f32(sign * gz(x00, y00))), f32(x00 - f32(sign * gz(x00, y11))), f32(x11 - f32(sign * gz(x11, y00)))]  # :714-719
    sy = [y00, y11, y00]
    v = f32(plane[3])
    if v != 0:                                     # (:720-725)
        sy = [f32(t + v) for t in sy]
    dx = [0.0, 0.0, float(f32(x11 - x00))]         # dst_pnt (:711-713)
    dy = [0.0, float(f32(y11 - y00)), 0.0]
    a = [[0.0] * 7 for _ in range(6)]
    for i in range(3):
        a[i] = [float(sx[i]), float(sy[i]), 1.0, 0.0, 0.0, 0.0, dx[i]]
        a[i + 3] = [0.0, 0.0, 0.0, float(sx[i]), float(sy[i]), 1.0, dy[i]]
    M = [0.0] * 6
    singular = False
    for c in range(6):
        piv = c
        for r in range(c + 1, 6):
            if abs(a[r][c]) > abs(a[piv][c]):
                piv = r
        if abs(a[piv][c]) < 2.220446049250313e-16:
            singular = True
            break
        if piv != c:
            a[c], a[piv] = a[piv], a[c]
        d = -1.0 / a[c][c]
        for r in range(c + 1, 6):
            f = a[r][c] * d
            for k in range(c + 1, 7):
                a[r][k] = a[r][k] + f * a[c][k]
    if not singular:
        for r in range(5, -1, -1):
            s = a[r][6]
            for k in range(r + 1, 6):
                s = s - a[r][k] * M[k]
            M[r] = s / a[r][r]
    D = M[0] * M[4] - M[1] * M[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[4] * D, M[0] * D
    i0, i1, i3, i4 = A11, M[1] * (-D), M[3] * (-D), A22
    i2 = (-i0) * M[2] - i1 * M[5]
    i5 = (-i3) * M[2] - i4 * M[5]
    return np.array([i0, i1, i2, i3, i4, i5], dtype=np.float64)


def warp_affine_linear_replicate(src, iM, w, h):
    """cv::warpAffine(src, dst, M, Size(w,h), INTER_LINEAR, BORDER_REPLICATE) for a float image with `iM` the
    already-inverted matrix: 10-bit fixed-point coordinates, 1/32-pixel bilinear weights."""
    H, W = src.shape[:2]
    xs = np.arange(w)
    ys = np.arange(h)
    adelta = _cv_round(iM[0] * xs * 1024.0)
    bdelta = _cv_round(iM[3] * xs * 1024.0)
    X0 = _cv_round((iM[1] * ys + iM[2]) * 1024.0) + 16
    Y0 = _cv_round((iM[4] * ys + iM[5]) * 1024.0) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx, sy = X >> 5, Y >> 5
    fx = ((X & 31).astype(np.float32) * f32(1.0 / 32)).astype(np.float32)
    fy = ((Y & 31).astype(np.float32) * f32(1.0 / 32)).astype(np.float32)
    w00 = ((f32(1) - fy) * (f32(1) - fx)).astype(np.float32)
    w01 = ((f32(1) - fy) * fx).astype(np.float32)
    w10 = (fy * (f32(1) - fx)).astype(np.float32)
    w11 = (fy * fx).astype(np.float32)
    x0c, x1c = np.clip(sx, 0, W - 1), np.clip(sx + 1, 0, W - 1)
    y0c, y1c = np.clip(sy, 0, H - 1), np.clip(sy + 1, 0, H - 1)
    S = src.reshape(H, W, -1)
    out = (S[y0c, x0c] * w00[..., None]).astype(np.float32)
    out = (out + S[y0c, x1c] * w01[..., None]).astype(np.float32)
    out = (out + S[y1c, x0c] * w10[..., None]).astype(np.float32)
    out = (out + S[y1c, x1c] * w11[..., None]).astype(np.float32)
    return out.reshape((h, w) + src.shape[2:])


class NaiveStereoEnergyOracle:
    """NaiveStereoEnergy (StereoEnergy.h:629-764), filterName "GF"."""

    def __init__(self, imL, imR, windR, eps, th_col, th_grad, alpha, max_disp, min_disp=0.0, box=box_sum_fast):
        self.im = [np.asarray(imL), np.asarray(imR)]
        self.windR, self.MAX, self.MIN = int(windR), f32(max_disp), f32(min_disp)
        self.ExI = [build_exI(self.im[0], alpha), build_exI(self.im[1], alpha)]
        self.thresh_color = f32(f32(th_col) * f32(f32(1.0) - f32(alpha)))   # :663
        self.thresh_gradient = f32(f32(th_grad) * f32(alpha))               # :664
        self.filter = [GuidedFilterStats(self.im[m], self.windR // 2, eps, np.float64, box=box) for m in range(2)]  # :674-675

    def raw(self, filter_rect, plane, mode=0):
        x, y, w, h = filter_rect
        iM = affine_inverse_for_plane(filter_rect, plane, mode)
        pIR = warp_affine_linear_replicate(self.ExI[1 - mode], iM, w, h)  # :729
        pIL = self.ExI[mode][y:y + h, x:x + w]
        d = np.abs(pIL - pIR).astype(np.float32)
        col = ((d[:, :, 0] + d[:, :, 1]).astype(np.float32) + d[:, :, 2]).astype(np.float32)
        return (np.minimum(self.thresh_color, col) + np.minimum(self.thresh_gradient, d[:, :, 3])).astype(np.float32)  # :737-740

    def compute_unary_potential_without_check(self, filter_rect, target_rect, plane, mode=0):
        p = self.raw(filter_rect, plane, mode)
        fx, fy, _, _ = filter_rect
        tx, ty, tw, th = target_rect
        q = guided_filter_sub(self.filter[mode], filter_rect, p)
        return q[ty - fy:ty - fy + th, tx - fx:tx - fx + tw].copy()

    def compute_unary_potential(self, filter_rect, target_rect, plane, mode=0):
        out = self.compute_unary_potential_without_check(filter_rect, target_rect, plane, mode)
        out[~is_valid_label(plane, target_rect, self.MIN, self.MAX)] = COST_FOR_INVALID  # :756-763
        return out


# ----------------------------------------------------------------------------
# PatchMatch phase: FastGCStereo::run's pmInit iterations = localExpansionMovesForLayer_CPU with doGC == false
# (FastGCStereo.h:22-72, 94-157).  Restated per proposal step so that it can be compared with the device path
# (lexp_plan_pm_step) launch by launch; pinned against the compiled reference's own loop (oracle/_ref ref_pm_group).
# ----------------------------------------------------------------------------
def pm_rng_state(seed, cell_id):
    """Start state of the cv::RNG stream of one (launch seed, cell): splitmix64 finaliser (= lexp::pm_rng_state)."""
    M = 0xFFFFFFFFFFFFFFFF
    z = (int(seed) + 0x9E3779B97F4A7C15 * ((int(cell_id) + 1) & 0xFFFFFFFF)) & M
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
    z = z ^ (z >> 31)
    return z if z else 0xFFFFFFFF


def pm_proposal(kind, m, state, cur_label, unit, min_disp, max_disp):
    """kind 1: ExpansionProposer::getNextProposal (Proposer.h:69-75); kind 2: RandomProposer::getNextProposal (:120-148);
    kind 3: RansacProposer(1) (:155-312, oracle/ransac_oracle.py)."""
    if kind == 3:
        from .ransac_oracle import ransac_proposal   # it imports this module for CvRNG
        return ransac_proposal(state, cur_label, unit)[0]
    rng = CvRNG(state)
    ux, uy, uw, uh = unit
    n = rng.uniform_int(0, uw * uh)                 # selectRandomPixelInRect (:38-45)
    sx, sy = ux + n % uw, uy + n // uw
    label = np.array(cur_label[sy, sx], dtype=np.float32)
    if kind == 1:
        return label
    return random_proposal(rng, label, sx, sy, m, min_disp, max_disp)


def pm_step(energy, units, shareds, filts, kind, m, seed, cell_ids, cur_cost, cur_label, planes=None, mode=0, init=False):
    """One proposal step for the (disjoint) cells of a group: proposal, ComputeUnaryPotential, `mask = cur > prop`, copy, setTo
    (FastGCStereo.h:47-59).  init: unconditional write (initCurrentFast, :107-111).  Returns the planes that were evaluated."""
    used = np.zeros((len(units), 4), np.float32)
    for i, (u, t, f) in enumerate(zip(units, shareds, filts)):
        if kind == 0:
            pl = np.asarray(planes[i], dtype=np.float32)
        else:
            pl = pm_proposal(kind, m, pm_rng_state(seed, cell_ids[i]), cur_label, u, energy.MIN, energy.MAX)
        used[i] = pl
        q = energy.compute_unary_potential(f, t, pl, mode)
        sl = (slice(t[1], t[1] + t[3]), slice(t[0], t[0] + t[2]))
        mask = np.ones(q.shape, bool) if init else (cur_cost[sl] > q)
        cur_cost[sl][mask] = q[mask]
        cur_label[sl][mask] = pl
    return used


# ---------------------------------------------------------------------------------------------------------------------
# Pairwise terms and the expansion move (SURVEY.md section 8 f-2 / f-3)
# ---------------------------------------------------------------------------------------------------------------------
NEIGHBORS = [(-1, 0), (1, 0), (0, -1), (0, 1), (-1, -1), (1, -1), (-1, 1), (1, 1)]   # StereoEnergy.h:100-110 (NB_LE .. NB_GG)
FORWARD = [1, 3, 6, 7]   # NB_GE, NB_EG, NB_LG, NB_GG: the neighbours with n.y * width + n.x > 0 (StereoEnergy.h:421)


def _shifted(a, dx, dy, fill=0):
    """b[y, x] = a[y + dy, x + dx], `fill` where that lies outside (a view of a zero-margined copy, StereoEnergy.h:136-143)."""
    H, W = a.shape[:2]
    m = np.full((H + 2, W + 2) + a.shape[2:], fill, a.dtype)
    m[1:-1, 1:-1] = a
    return m[1 + dy:1 + dy + H, 1 + dx:1 + dx + W]


def smoothness_coeff(im8, omega=10.0, epsilon=0.01):
    """StereoEnergy::initSmoothnessCoeff (StereoEnergy.h:131-163) without the margin: float32 [8][H][W].
    coeff_k = max(epsilon, exp(-channelSum(|I(p + n_k) - I(p)|) / omega)), zero where p + n_k is outside the image."""
    I = np.asarray(im8).astype(np.float32)
    H, W = I.shape[:2]
    out = np.zeros((8, H, W), np.float32)
    xs, ys = np.meshgrid(np.arange(W), np.arange(H))
    for k, (dx, dy) in enumerate(NEIGHBORS):
        d = np.abs(_shifted(I, dx, dy) - I)                               # absdiff (:144)
        s = (d[..., 0] + d[..., 1]) + d[..., 2]                           # channelSum (Utilities.hpp:224-229)
        c = np.exp((s * np.float32(-1.0)).astype(np.float64) * (1.0 / float(omega))).astype(np.float32)   # -m / omega as MatExpr: scale in double (:145)
        c = np.maximum(np.float32(epsilon), c)                            # :146
        inside = (xs + dx >= 0) & (xs + dx < W) & (ys + dy >= 0) & (ys + dy < H)
        out[k] = np.where(inside, c, np.float32(0))                       # :148-156
    return out


def _disp(lab, X, Y):
    """cvutils::channelDot(label, coord) with coord = (x, y, 1, 0): the 4-term row sum in float (Utilities.hpp:215-222)."""
    a, b, c, v = (lab[..., i].astype(np.float32) for i in range(4))
    X, Y = np.float32(X) if np.isscalar(X) else X.astype(np.float32), np.float32(Y) if np.isscalar(Y) else Y.astype(np.float32)
    return ((a * X + b * Y) + c) + v * np.float32(0)


def smoothness_terms_expansion(labeling, plane, region, coeff, lam=1.0, th_smooth=1.0):
    """StereoEnergy::computeSmoothnessTermsExpansion(labeling0_m, label1, region, .., onlyForward = true) (StereoEnergy.h:398-453).
    labeling float32 [H][W][4] (its margin is zero, PMStereoBase.h:44), coeff = smoothness_coeff(..)[8][H][W].
    Returns cost00, cost01, cost10: float32 [8][h][w], filled for the forward neighbours only."""
    lab = np.asarray(labeling, np.float32)
    H, W = lab.shape[:2]
    x0, y0, w, h = (int(v) for v in region)
    l1 = np.asarray(plane, np.float32).reshape(1, 1, 4)
    lam, th = np.float32(lam), np.float32(th_smooth)
    xs, ys = np.meshgrid(np.arange(x0, x0 + w), np.arange(y0, y0 + h))
    sl = (slice(y0, y0 + h), slice(x0, x0 + w))
    L_ee = lab[sl]
    d0_ee_ee = _disp(L_ee, xs, ys)                                        # :405
    d1_ee = _disp(l1, xs, ys)                                             # :406
    c00, c01, c10 = (np.zeros((8, h, w), np.float32) for _ in range(3))
    for k in FORWARD:
        dx, dy = NEIGHBORS[k]
        inside = (xs + dx >= 0) & (xs + dx < W) & (ys + dy >= 0) & (ys + dy < H)
        L_le = _shifted(lab, dx, dy)[sl]                                  # zero label in the margin
        qx, qy = np.where(inside, xs + dx, 0), np.where(inside, ys + dy, 0)
        one = inside.astype(np.float32)                                   # coordinates_m is (x, y, 1, 0) inside, zero in the margin

        def disp_at_le(L):
            a, b, c, v = (L[..., i].astype(np.float32) for i in range(4))
            return ((a * qx.astype(np.float32) + b * qy.astype(np.float32)) + c * one) + v * np.float32(0)
        d0_le_ee = _disp(L_le, xs, ys)                                    # :426
        d0_ee_le = disp_at_le(L_ee)                                       # :427
        d0_le_le = disp_at_le(L_le)                                       # :428
        d1_le = disp_at_le(np.broadcast_to(l1, L_ee.shape))               # :429
        co = coeff[k][sl]

        def term(a0, a1, b0, b1):
            c = np.abs(a0 - a1) + np.abs(b0 - b1)
            c = np.where(c > th, th, c)                                   # THRESH_TRUNC
            return (lam * c) * co                                         # Mat::mul(coeff, lambda)
        c00[k] = term(d0_ee_ee, d0_le_ee, d0_ee_le, d0_le_le)             # :441-443
        c01[k] = term(d0_ee_ee, d1_ee, d0_ee_le, d1_le)                   # :445-447
        c10[k] = term(d1_ee, d0_le_ee, d1_le, d0_le_le)                   # :449-451
    return c00, c01, c10


def _get_z(lab, X, Y):
    """Plane::GetZ(cv::Point) = a x + b y + c (Plane.h:55-58)."""
    a, b, c = (lab[..., i].astype(np.float32) for i in range(3))
    return (a * np.float32(X) + b * np.float32(Y)) + c


def smoothness_term(ls, lt, ps, k, coeff, lam, th_smooth):
    """StereoEnergy::computeSmoothnessTerm(ls, lt, ps, neighborId, mode) (StereoEnergy.h:234-239)."""
    pt = (ps[0] + NEIGHBORS[k][0], ps[1] + NEIGHBORS[k][1])
    ls, lt = np.asarray(ls, np.float32), np.asarray(lt, np.float32)
    s = np.abs(_get_z(ls, *ps) - _get_z(lt, *ps)) + np.abs(_get_z(ls, *pt) - _get_z(lt, *pt))
    return (np.float32(coeff[k][ps[1], ps[0]]) * np.minimum(np.float32(s), np.float32(th_smooth))) * np.float32(lam)


def expansion_graph(cur_cost, cur_label, prop_cost, plane, region, coeff, lam=1.0, th_smooth=1.0):
    """The graph FastGCStereo::expansionMoveBK builds (FastGCStereo.h:424-549) for the move `plane` on `region`: returns
    (tr, konst, cap): tr float32 [h][w] = the NET terminal capacity of every node as the BK library holds it after the reference's
    sequence of Graph::add_tweights calls (float, the same operations in the same order), konst = the part of the flow value those
    calls add (`flow += min(cap_source, cap_sink)`), cap float32 [4][h][w] = capacities of the forward arcs (GE, EG, LG, GG)."""
    x0, y0, w, h = (int(v) for v in region)
    H, W = cur_cost.shape
    sl = (slice(y0, y0 + h), slice(x0, x0 + w))
    c00, c01, c10 = smoothness_terms_expansion(cur_label, plane, region, coeff, lam, th_smooth)   # :422
    tr = np.zeros((h, w), np.float32)
    konst = np.zeros((h, w), np.float64)

    def add_tweights(sel, cap_source, cap_sink):   # Graph::add_tweights, element-wise on the nodes `sel`
        nonlocal tr, konst
        cs = np.where(tr > 0, (cap_source + tr).astype(np.float32), cap_source).astype(np.float32)
        ck = np.where(tr > 0, cap_sink, (cap_sink - tr).astype(np.float32)).astype(np.float32)
        konst = np.where(sel, konst + np.minimum(cs, ck).astype(np.float64), konst)
        tr = np.where(sel, (cs - ck).astype(np.float32), tr)
    every = np.ones((h, w), bool)
    q = np.asarray(prop_cost, np.float32)
    assert q.shape == (h, w)
    with np.errstate(invalid="ignore"):
        add_tweights(every, cur_cost[sl].astype(np.float32), q)               # :433
    l1 = np.asarray(plane, np.float32)
    ys, xs = np.mgrid[0:h, 0:w]
    for k, (dx, dy) in enumerate(NEIGHBORS):                                  # outer boundary (:435-471), reference neighbour order
        a = np.zeros((h, w), np.float32); b = np.zeros((h, w), np.float32); sel = np.zeros((h, w), bool)
        for y in range(h):
            for x in (range(w) if y in (0, h - 1) else sorted({0, w - 1})):
                ps = (x0 + x, y0 + y)
                pt = (ps[0] + dx, ps[1] + dy)
                if x0 <= pt[0] < x0 + w and y0 <= pt[1] < y0 + h:
                    continue
                if not (0 <= pt[0] < W and 0 <= pt[1] < H):
                    continue
                lt = cur_label[pt[1], pt[0]]
                a[y, x] = smoothness_term(cur_label[ps[1], ps[0]], lt, ps, k, coeff, lam, th_smooth)
                b[y, x] = smoothness_term(l1, lt, ps, k, coeff, lam, th_smooth)
                sel[y, x] = True
        add_tweights(sel, a, b)
    cap = np.zeros((4, h, w), np.float32)
    zero = np.zeros((h, w), np.float32)
    for fi, k in enumerate([1, 3, 6, 7]):                                     # GE, EG, LG, GG (:478-541)
        dx, dy = NEIGHBORS[k]
        B, C_, D = c10[k], c01[k], c00[k]
        ok = (xs + dx >= 0) & (xs + dx < w) & (ys + dy < h)                   # pairs (i, j = i + n) inside the region
        cap[fi] = np.where(ok, np.maximum(np.float32(0), (B + C_) - D), np.float32(0))   # add_edge(i, j, max(0, B + C - D), 0)
        DmC = np.zeros((h, w), np.float32); is_j = np.zeros((h, w), bool)     # the pair's values moved to its node j
        DmC[max(dy, 0):h, max(dx, 0):w + min(dx, 0)] = (D - C_)[0:h - max(dy, 0), max(-dx, 0):w - max(dx, 0)]
        is_j[max(dy, 0):h, max(dx, 0):w + min(dx, 0)] = ok[0:h - max(dy, 0), max(-dx, 0):w - max(dx, 0)]
        add_tweights(is_j, DmC, zero)                                         # add_tweights(j, D - C, 0): reached before the node's own pair
        add_tweights(ok, C_, zero)                                            # add_tweights(i, C, 0)
    return tr, float(konst.sum()), cap


def expansion_move(cur_cost, cur_label, prop_cost, plane, region, coeff, lam=1.0, th_smooth=1.0):
    """FastGCStereo::expansionMoveBK (FastGCStereo.h:411-597): (updateMask bool [h][w], flow as BK reports it)."""
    from . import c_oracle
    tr, konst, cap = expansion_graph(cur_cost, cur_label, prop_cost, plane, region, coeff, lam, th_smooth)
    mask, mf = c_oracle.grid_mincut(tr, cap)
    return mask, konst + mf


def gc_step(energy, units, shareds, filts, kind, m, seed, cell_ids, cur_cost, cur_label, coeff, lam=1.0, th_smooth=1.0, planes=None, mode=0):
    """One proposal step with doGC == true for the (disjoint) cells of a group: proposal, ComputeUnaryPotential, expansionMoveBK,
    copyTo / setTo (FastGCStereo.h:47-59).  Returns (planes evaluated [n][4], flows [n])."""
    used = np.zeros((len(units), 4), np.float32)
    flows = np.zeros(len(units), np.float64)
    for i, (u, t, f) in enumerate(zip(units, shareds, filts)):
        if kind == 0:
            pl = np.asarray(planes[i], dtype=np.float32)
        else:
            pl = pm_proposal(kind, m, pm_rng_state(seed, cell_ids[i]), cur_label, u, energy.MIN, energy.MAX)
        used[i] = pl
        q = energy.compute_unary_potential(f, t, pl, mode)
        mask, flows[i] = expansion_move(cur_cost, cur_label, q, pl, t, coeff, lam, th_smooth)
        sl = (slice(t[1], t[1] + t[3]), slice(t[0], t[0] + t[2]))
        cur_cost[sl][mask] = q[mask]
        cur_label[sl][mask] = pl
    return used, flows


def smoothness_cost(labeling, coeff, lam=1.0, th_smooth=1.0):
    """StereoEnergy::computeSmoothnessCost (StereoEnergy.h:165-199): sum over the forward neighbour pairs of the image."""
    lab = np.asarray(labeling, np.float32)
    H, W = lab.shape[:2]
    c00, _, _ = smoothness_terms_expansion(lab, np.zeros(4, np.float32), (0, 0, W, H), coeff, lam, th_smooth)
    return float(sum(c00[k].astype(np.float64).sum() for k in FORWARD))
