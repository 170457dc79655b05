"""(Runs last in the -m gpu suite, with tests/test_gpu_zzz_sizes.py: it allocates the most device memory.)

The bilateral filter ("BL") and the unfiltered mode ("") of the cost-volume energy at the 4K stress case 3840 x 2160 x 512, windR 32
(BASELINE.json configs[4]): the blocked volume holds 4.2e9 elements (17 GB), so the offsets of lc_raw_volume pass 2^31 elements and
only size_t arithmetic reads the right cost.  Sampled cells of layer 0 and layer 2 -- always the bottom-right border cell, whose
block offset is the largest, and the largest filterRect -- against per-cell oracles built from host slabs of the volume, with and without the check:
"" bit for bit on the whole targetRect, so a wrapped offset cannot hide behind a tolerance; "BL" within 1e-5 max(sum w |p|, 1e-3) on
the targetRect's top-left and bottom-right 48 x 48 corners; the NaN and COST_FOR_INVALID patterns exactly."""
import time

import numpy as np
import pytest

from oracle import lexp_oracle as O
from oracle.filter_oracle import bilateral_sub
from test_gpu_golden import _OffsetVolume

pytestmark = pytest.mark.gpu

SIG2 = 10.0


def _oracle_rects(img, slab, f, t, p, filt, windR, D, with_check, th=0.5):
    """[(rect, q, sum w |p|)] of the call (f, t, p) from the filterRect slab of the volume: the whole targetRect for "", its two
    corners for "BL"."""
    raw = O.sample_plane_cost(_OffsetVolume(slab, f[0], f[1]), f, p, np.float32(th), 0.0, D - 1)
    x, y, w, h = t
    if filt == "":
        rects = [tuple(t)]
    else:
        c = 48
        rects = [(x, y, min(c, w), min(c, h)), (x + w - min(c, w), y + h - min(c, h), min(c, w), min(c, h))]
    out = []
    for r in rects:
        rx, ry, rw, rh = r
        if filt == "":
            q = raw[ry - f[1]:ry - f[1] + rh, rx - f[0]:rx - f[0] + rw].astype(np.float64)
            s = np.abs(q)
        else:
            q, s = bilateral_sub(img, f, r, raw, windR, float(np.float32(SIG2)))
        if with_check:
            bad = ~O.is_valid_label(p, t, 0.0, D - 1)[ry - y:ry - y + rh, rx - x:rx - x + rw]
            q[bad] = O.COST_FOR_INVALID
            s[bad] = O.COST_FOR_INVALID
        out.append((r, q, s))
    return out


@pytest.mark.parametrize("filt", ["", "BL"])
def test_4k_sampled_cells_of_layers_0_and_2(filt):
    import torch
    import localexpstereo_b200 as L
    import filter_checks as FC
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import v3_layer_units
    W, H, D, windR = 3840, 2160, 512, 32
    t0 = time.perf_counter()
    vol = torch.rand((D, H, W), generator=torch.Generator(device="cuda").manual_seed(99), device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()   # torch fills the volume on its own stream; the library's stream is non-blocking
    img = synth.synthetic_image(H, W, 42)
    prm = L.Parameters(windR=windR, filterName=filt, filter_param1=SIG2, th_col=0.5)
    E = L.CostVolumeEnergy(img, None, vol, None, prm, D - 1)
    try:
        lm = L.LayerManager(W, H, windR)
        rng = np.random.default_rng(29)
        worst, n_cells, n_corner = 0.0, 0, 0
        units = v3_layer_units(W)
        for li in range(3):
            lay = lm.addLayer(units[li])
            if li == 1:
                continue
            corner = next(r for r, (x, y, w, h) in enumerate(lay.sharedRegions) if (x + w, y + h) == (W, H))
            grp = next(g for g in lay.disjointRegionSets if corner in g)
            planes = synth.synthetic_planes(lay.unitRegions, 2, D, 11 + li)[1][grp]
            fr = np.array([lay.filterRegions[r] for r in grp], np.int32)
            tr = np.array([lay.sharedRegions[r] for r in grp], np.int32)
            P = E.make_plan(fr, tr)
            outs = {}
            for wc in (True, False):
                outs[wc] = np.full((H, W), -1.0, np.float32)
                P.eval_host(planes, outs[wc], with_check=wc)
            P.close()
            big = int(np.argmax(fr[:, 2].astype(np.int64) * fr[:, 3]))
            pick = {list(grp).index(corner), big} | set(int(i) for i in rng.choice(len(grp), size=1))
            for i in sorted(pick):
                f, t, p = fr[i], tr[i], planes[i]
                slab = vol[:, f[1]:f[1] + f[3], f[0]:f[0] + f[2]].cpu().numpy()
                for wc in (True, False):
                    for (rx, ry, rw, rh), q, s in _oracle_rects(img, slab, f, t, p, filt, windR, D, wc):
                        worst = max(worst, FC.compare(outs[wc][ry:ry + rh, rx:rx + rw], q, s, filt == "",
                                                      f"{filt!r} 4K layer {li} cell {grp[i]} rect {(rx, ry, rw, rh)} check {wc}"))
                del slab
                n_cells += 1
                n_corner += int(grp[i] == corner)
        assert n_corner == 2
        print(f"{filt!r} 3840 x 2160 x 512 r32: {n_cells} cells of layers 0 and 2, worst |d| / sum w|p| {worst:.2e}; "
              f"{time.perf_counter() - t0:.1f} s")
    finally:
        E.close()
        del vol
        torch.cuda.empty_cache()
