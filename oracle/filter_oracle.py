"""FP64 restatement of the reference's two other aggregation filters, on top of the raw costs of oracle/lexp_oracle.py:

  BilateralFilter::filter (GuidedFilter.h:329-373) -- filterName "BL" for CostVolumeEnergy (CostVolumeEnergy.h:25-28), "BF" for
  NaiveStereoEnergy (StereoEnergy.h:668-671):
      q(x) = sum over y in (x +- windR) & filterRect of p(y) exp(-(|I0(y)-I0(x)| + |I1(y)-I1(x)| + |I2(y)-I2(x)|) / sig2)
  with radius windR (the BilateralFilter gets params.windR, the guided filter windR / 2), the 8-bit BGR guide as float, unscaled
  (:348-349), sig2 = filter_param1, the window clipped at the filterRect (createSubregionFilter hands the filter I(rect), :352-355)
  and the sum not normalised (:365);
  filterName "": the raw cost itself (CostVolumeEnergy.h:169-171, StereoEnergy.h:752-753).
Then ComputeUnaryPotential's validity mask (CostVolumeEnergy.h:176-182, StereoEnergy.h:756-763).

The weights and the sum are evaluated in FP64.  `unary` also returns sum w |p| per pixel: the scale of the float rounding of the
reference (float exp, float weights) and of the device (float weights, float sums), against which the tests set their tolerance."""
import numpy as np

from .lexp_oracle import COST_FOR_INVALID, CostVolumeEnergyOracle, NaiveStereoEnergyOracle, is_valid_label


def bilateral_sub(im8, filter_rect, target_rect, p, windR, sig2):
    """q and sum w |p| (float64 [th][tw]) of BilateralFilter(I(filterRect), windR, sig2).filter(p) on targetRect; p = raw costs
    float32 [fh][fw] of the filterRect."""
    fx, fy, fw, fh = filter_rect
    tx, ty, tw, th = target_rect
    I = np.asarray(im8).astype(np.int64)
    P = np.asarray(p, np.float64)
    ys = np.arange(ty, ty + th)[:, None]
    xs = np.arange(tx, tx + tw)[None, :]
    Ic = I[ty:ty + th, tx:tx + tw]
    q = np.zeros((th, tw))
    scale = np.zeros((th, tw))
    with np.errstate(invalid="ignore", over="ignore"):
        for dy in range(-windR, windR + 1):
            yy = ys + dy
            oky = (yy >= fy) & (yy < fy + fh)
            yyc = np.clip(yy, fy, fy + fh - 1)
            for dx in range(-windR, windR + 1):
                xx = xs + dx
                ok = oky & (xx >= fx) & (xx < fx + fw)
                if not ok.any():
                    continue
                xxc = np.clip(xx, fx, fx + fw - 1)
                s = np.abs(I[yyc, xxc] - Ic).sum(-1)                         # channelSum(|I(patch) - I(x)|) (:362)
                w = np.exp(-s / float(sig2))                                 # (:363)
                pv = P[yyc - fy, xxc - fx]
                q += np.where(ok, pv * w, 0.0)                               # p(patch).dot(w) (:365)
                scale += np.where(ok, np.abs(pv) * w, 0.0)
    return q, scale


class FilteredEnergyOracle:
    """A CostVolumeEnergy ("BL" / "") or NaiveStereoEnergy ("BF" / "") of the reference.  `base` supplies the raw costs (its
    `raw(filterRect, plane, mode)`), `im` the two guides."""

    def __init__(self, base, im, windR, sig2, bilateral):
        self.base, self.im = base, im
        self.windR, self.sig2, self.bilateral = int(windR), float(np.float32(sig2)), bool(bilateral)
        self.MIN, self.MAX = base.MIN, base.MAX

    @staticmethod
    def cost_volume(imL, imR, volL, volR, windR, sig2, th_col, max_disp, min_disp=0.0, bilateral=True):
        base = CostVolumeEnergyOracle(imL, imR, volL, volR, windR, sig2, th_col, max_disp, min_disp, filter_name="")
        return FilteredEnergyOracle(base, [imL, imR], windR, sig2, bilateral)

    @staticmethod
    def naive(imL, imR, windR, sig2, th_col, th_grad, alpha, max_disp, min_disp=0.0, bilateral=True):
        base = NaiveStereoEnergyOracle(imL, imR, windR, 1e-4, th_col, th_grad, alpha, max_disp, min_disp)
        return FilteredEnergyOracle(base, [imL, imR], windR, sig2, bilateral)

    def unary(self, filter_rect, target_rect, plane, mode=0, with_check=True):
        """(q, scale), float64 [th][tw]: ComputeUnaryPotential[WithoutCheck] on targetRect and sum w |p| (|q| for "")."""
        p = self.base.raw(filter_rect, plane, mode)
        fx, fy, _, _ = filter_rect
        tx, ty, tw, th = target_rect
        if self.bilateral:
            q, scale = bilateral_sub(self.im[mode], filter_rect, target_rect, p, self.windR, self.sig2)
        else:
            q = p[ty - fy:ty - fy + th, tx - fx:tx - fx + tw].astype(np.float64)
            scale = np.abs(q)
        if with_check:
            bad = ~is_valid_label(plane, target_rect, self.MIN, self.MAX)
            q[bad] = COST_FOR_INVALID
            scale[bad] = COST_FOR_INVALID
        return q, scale

    def compute_unary_potential(self, filter_rect, target_rect, plane, mode=0):   # the interface of lexp_oracle.pm_step
        return self.unary(filter_rect, target_rect, plane, mode)[0]
