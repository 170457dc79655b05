"""numpy restatement of PMStereoBase::postProcess (PMStereoBase.h:146-256) and doConsistencyCheck (:111-144): the oracle of
tests/test_*_post.py.  Float arithmetic as in the reference: computeDisparities = channelDot((x, y, 1, 0), L) and Plane::GetZ with every
product and sum rounded separately in float32; weights exp(-absdiff / omega) from the C library's expf (numpy's float32 exp is a
different implementation); both sums of the weights sequential in float64 (np.cumsum, never the pairwise np.sum).

The reference leaves the order of equal median keys to std::sort.  Here, as on the device, candidates are ordered by (key, row-major
index in the window), -0 equal to +0 and NaN after every number; `post_process` also reports the pixels whose chosen key is tied with
another candidate's, where the reference may pick a different plane of the same disparity."""
import ctypes
import ctypes.util

import numpy as np

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.expf.restype = ctypes.c_float
_libm.expf.argtypes = [ctypes.c_float]


def weight_table(omega):
    """computePatchWeight (StereoEnergy.h:251-257) for absdiff = 0 .. 765: std::exp(-absdiff / omega) in float."""
    om = np.float32(omega)
    return np.array([_libm.expf(float(np.float32(-k) / om)) for k in range(766)], np.float32)


def disparities(lab):
    """StereoEnergy::computeDisparities: lab [H][W][4] float32 -> [H][W] float32."""
    H, W = lab.shape[:2]
    x = np.arange(W, dtype=np.float32)[None, :]
    y = np.arange(H, dtype=np.float32)[:, None]
    with np.errstate(all="ignore"):
        return ((lab[..., 0] * x + lab[..., 1] * y) + lab[..., 2]) + lab[..., 3] * np.float32(0)


def getz(lab, x, y):
    """Plane::GetZ(x, y) = a x + b y + c for planes lab[..., 4] at float32 points x, y (broadcast)."""
    with np.errstate(all="ignore"):
        return (lab[..., 0] * np.float32(x) + lab[..., 1] * np.float32(y)) + lab[..., 2]


def consistency_check(lab0, lab1, threshold=1.5):
    """doConsistencyCheck(disp0, disp1, fail0, fail1, threshold): uint8 [2][H][W] of 0 / 255 (|dsr - ds| > threshold) / 128 (rx outside
    the image).  rx = int(x - ds * sign + 0.5f) as x86-64's cvttss2si: truncation toward zero, INT_MIN for NaN and |v| >= 2^31."""
    H, W = lab0.shape[:2]
    disp = [disparities(lab0), disparities(lab1)]
    xs = np.broadcast_to(np.arange(W, dtype=np.float32)[None, :], (H, W))
    ys = np.broadcast_to(np.arange(H)[:, None], (H, W))
    fail = np.zeros((2, H, W), np.uint8)
    thr = np.float32(threshold)
    with np.errstate(all="ignore"):
        for i in range(2):
            sign = np.float32(-1.0 if i else 1.0)
            v = (xs - disp[i] * sign) + np.float32(0.5)
            conv = np.isfinite(v) & (v > np.float32(-2147483648.0)) & (v < np.float32(2147483648.0))
            rx = np.where(conv, np.trunc(np.where(conv, v, 0)), -1).astype(np.int64)
            inside = conv & (rx >= 0) & (rx < W)
            dsr = disp[1 - i][ys, np.clip(rx, 0, W - 1)]
            bad = np.abs(dsr - disp[i]) > thr
            fail[i][inside & bad] = 255
            fail[i][~inside] = 128
    return fail


def dilate3x3(mask):
    """cv::dilate(mask, out, cv::Mat()) of a boolean map: 3x3 rectangle, pixels outside the image never contribute."""
    H, W = mask.shape
    p = np.zeros((H + 2, W + 2), bool)
    p[1:-1, 1:-1] = mask
    out = np.zeros((H, W), bool)
    for dy in range(3):
        for dx in range(3):
            out |= p[dy:dy + H, dx:dx + W]
    return out


def hole_fill(lab, fail):
    """The horizontal nearest-neighbour fill (:169-202) of one view: returns the filled copy of lab."""
    H, W = fail.shape
    fail2 = dilate3x3(fail > 0)
    idx = np.broadcast_to(np.arange(W)[None, :], (H, W))
    left = np.maximum.accumulate(np.where(~fail2, idx, -1), axis=1)
    right = np.minimum.accumulate(np.where(~fail2, idx, W)[:, ::-1], axis=1)[:, ::-1]
    out = lab.copy()
    ys, xs = np.nonzero(fail > 0)
    l, r = left[ys, xs], right[ys, xs]
    Ll, Lr = lab[ys, np.clip(l, 0, W - 1)], lab[ys, np.clip(r, 0, W - 1)]
    fx, fy = xs.astype(np.float32), ys.astype(np.float32)
    take_l = getz(Ll, fx, fy) < getz(Lr, fx, fy)
    both = (l >= 0) & (r < W)
    pick = np.where((both & take_l)[:, None] | ((l >= 0) & (r >= W))[:, None], Ll,
                    np.where((r < W)[:, None], Lr, lab[ys, xs]))
    out[ys, xs] = pick
    return out


def sort_keys(z):
    """uint32 keys whose order is the order of the float keys: -0 == +0, NaN after every number."""
    z = np.where(z == 0, np.float32(0), z).astype(np.float32)
    u = z.view(np.uint32)
    k = np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)
    k[np.isnan(z)] = np.uint32(0xFFFFFFFF)
    return k


def median_pixel(filled, im, x, y, windR, wtab):
    """The weighted median (:209-252) at (x, y) of one view: (chosen plane, its key is tied with another candidate's)."""
    H, W = filled.shape[:2]
    x0, x1, y0, y1 = max(x - windR, 0), min(x + windR + 1, W), max(y - windR, 0), min(y + windR + 1, H)
    cand = filled[y0:y1, x0:x1].reshape(-1, 4)
    g = im[y0:y1, x0:x1].reshape(-1, 3).astype(np.int32)
    ad = np.abs(g - im[y, x].astype(np.int32)).sum(axis=1)
    w = wtab[ad].astype(np.float64)
    center = np.cumsum(w)[-1] / 2.0
    keys = getz(cand, x, y)
    order = np.argsort(sort_keys(keys), kind="stable")
    run = np.cumsum(w[order])
    hit = np.nonzero(run > center)[0]
    if len(hit) == 0:
        return filled[y, x].copy(), False
    c = order[hit[0]]
    kc = keys[c]
    tied = int(np.count_nonzero(keys == kc)) > 1 if not np.isnan(kc) else True
    return cand[c].copy(), tied


def post_process(lab0, lab1, im0, im1, windR, omega, threshold=1.5, pixels=None):
    """PMStereoBase::postProcess(lab0, lab1, threshold) with params.windR = windR and params.omega = omega.  Returns (out0, out1, fail,
    tied) where fail is consistency_check's map and tied[i] a bool [H][W] map of the median pixels whose chosen key is tied.
    `pixels`: optional per-view lists of (y, x) failed pixels to run the median on (the others keep the filled label and are marked
    in the returned `done` maps); None = every failed pixel."""
    fail = consistency_check(lab0, lab1, threshold)
    wtab = weight_table(omega)
    outs, tied, done = [], [], []
    for i, (lab, im) in enumerate(((lab0, im0), (lab1, im1))):
        filled = hole_fill(lab, fail[i])
        out = lab.copy()
        t = np.zeros(lab.shape[:2], bool)
        d = np.zeros(lab.shape[:2], bool)
        todo = zip(*np.nonzero(fail[i] > 0)) if pixels is None else pixels[i]
        for y, x in todo:
            assert fail[i][y, x] > 0
            out[y, x], t[y, x] = median_pixel(filled, im, int(x), int(y), windR, wtab)
            d[y, x] = True
        outs.append(out)
        tied.append(t)
        done.append(d)
    return outs[0], outs[1], fail, tied, done
