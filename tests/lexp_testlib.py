"""Shared helpers for the parity tests: seeded synthetic scenes, contexts with their oracles, device memory and comparison rules."""
import contextlib
import os

import numpy as np

from oracle import lexp_oracle as O

REL_TOL = 1e-4      # north_star: "within 1e-4 relative float tolerance on aggregated costs"
ABS_FLOOR = 1e-3    # SURVEY.md 8(d): |delta| <= 1e-4 * max(|ref|, 1e-3)


def make_scene(H, W, D, seed=0, natural=None):
    img = natural if natural is not None else O.synthetic_image(H, W, 42 + seed)
    imgR = O.synthetic_image(H, W, 43 + seed) if natural is None else natural[:, ::-1].copy()
    volL = O.synthetic_volume(D, H, W, 1234 + seed)
    volR = O.synthetic_volume(D, H, W, 1235 + seed)
    return img, imgR, volL, volR


def assert_costs_close(got, ref, what=""):
    got = np.asarray(got)
    ref = np.asarray(ref)
    inv_ref = ref == O.COST_FOR_INVALID
    inv_got = got == O.COST_FOR_INVALID
    assert np.array_equal(inv_ref, inv_got), f"{what}: COST_FOR_INVALID mask differs at {np.argwhere(inv_ref != inv_got)[:5]}"
    ok = ~inv_ref
    if ok.any():
        err = np.abs(got[ok].astype(np.float64) - ref[ok].astype(np.float64))
        tol = REL_TOL * np.maximum(np.abs(ref[ok]), ABS_FLOOR)
        worst = float((err / tol).max())
        assert worst <= 1.0, f"{what}: max err/tol = {worst:.3f} (max abs err {err.max():.3e})"
        return worst * REL_TOL
    return 0.0


def random_planes(rng: O.CvRNG, units, D):
    out = []
    for (ux, uy, uw, uh) in units:
        n = rng.uniform_int(0, uw * uh)
        out.append(O.create_random_label(rng, ux + n % uw, uy + n // uw, 0.0, float(D - 1)))
    return np.stack(out)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def energy_and_oracle(scene, D, windR, mode=0, naive=False, **params):
    """A context on scene = (imL, imR, volL, volR) and the oracle of the same energy: the cost-volume energy (the right view's
    inputs only for mode = 1), or the image-based energy of -mode MiddV2 (naive).  params: further Parameters fields."""
    import localexpstereo_b200 as L
    imL, imR, volL, volR = scene
    if naive:
        prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, **params)
        return (L.NaiveStereoEnergy(imL, imR, prm, D - 1),
                O.NaiveStereoEnergyOracle(imL, imR, windR, 1e-4, prm.th_col, prm.th_grad, prm.alpha, D - 1))
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5, **params)
    imR, volR = (imR, volR) if mode else (None, None)
    return L.CostVolumeEnergy(imL, imR, volL, volR, prm, D - 1), O.CostVolumeEnergyOracle(imL, imR, volL, volR, windR, 1e-4, prm.th_col, D - 1)


def seeded_labels(S, seed):
    """Initial labels of the sweep S's layer-0 units: a random plane through a random pixel of each unit (O.CvRNG(seed))."""
    rng = O.CvRNG(seed)
    lo, hi = S.energy.MIN_DISPARITY, S.energy.MAX_DISPARITY
    return np.stack([O.create_random_label(rng, u[0] + rng.uniform_int(0, u[2]), u[1] + rng.uniform_int(0, u[3]), lo, hi) for u in S.init_units])


@contextlib.contextmanager
def pdl_off():
    """Contexts created inside launch every kernel stream-serialised (lexp_create reads LEXP_PDL_OFF)."""
    prev = os.environ.get("LEXP_PDL_OFF")
    os.environ["LEXP_PDL_OFF"] = "1"
    try:
        yield
    finally:
        if prev is None:
            os.environ.pop("LEXP_PDL_OFF")
        else:
            os.environ["LEXP_PDL_OFF"] = prev


class TorchDeviceMemory:
    """Device buffers for the device-output entry points: torch CUDA tensors on the GPU."""

    def __init__(self):
        import torch
        self.torch = torch

    # the context launches on its own non-blocking stream: buffers must be complete before their pointers are handed over
    def zeros(self, shape, fill=0.0):
        t = self.torch.full(shape, fill, dtype=self.torch.float32, device="cuda")
        self.torch.cuda.synchronize()
        return t

    def upload(self, a):
        t = self.torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.torch.cuda.synchronize()
        return t

    @staticmethod
    def ptr(t):
        return t.data_ptr()

    def download(self, t):
        self.torch.cuda.synchronize()
        return t.cpu().numpy()


class HostAsDeviceMemory:
    """On the emulator device memory is host memory: numpy arrays stand in for the device buffers."""

    @staticmethod
    def zeros(shape, fill=0.0):
        return np.full(shape, fill, np.float32)

    @staticmethod
    def upload(a):
        return np.ascontiguousarray(a)

    @staticmethod
    def ptr(t):
        return t.ctypes.data

    @staticmethod
    def download(t):
        return t
