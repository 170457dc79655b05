"""Times lexp_pm_init_from_labeling (initCurrentFast started from a given labeling, FastGCStereo.h:116-130) against the routes that
existed before it, and prints one JSON line per measurement:
  * the new call on the whole image: 2048 x 1536 x 256 at windR 20 and 960 x 544 x 96 at windR 32, both energy kinds, on two plane
    fields -- the labeling of a device run (initialisation + one pm iteration of the cost-volume energy: piecewise smooth) and
    independent random planes per pixel (the worst case for locality);
  * the best existing route: one plan of 1x1-target calls (filterRect F(p)) through lexp_plan_eval_device on a band of rows, per pixel;
  * the compiled reference's own branch (ref_pm_init with 1x1 units, 16 host threads) on a crop, per pixel, where oracle/_ref is built.
CUDA events around each device call (median of the repetitions after warm-up).  Usage: python scripts/label_cost_bench.py [--quick]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def timed(fn, stream, warmup=2, reps=5):
    import torch
    s = torch.cuda.ExternalStream(stream)
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        fn()
        b.record(s)
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def main():
    import torch
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import PMSweep
    import label_cost_checks as LC
    from lexp_testlib import seeded_labels
    quick = "--quick" in sys.argv
    gpu, power = card()
    configs = [(2048, 1536, 256, 20), (960, 544, 96, 32)]
    for (W, H, D, windR) in configs:
        imL, imR = synth.synthetic_image(H, W, 42), synth.synthetic_image(H, W, 43)
        vol = torch.rand((D, H, W), generator=torch.Generator(device="cuda").manual_seed(1234), device="cuda", dtype=torch.float32)
        torch.cuda.synchronize()
        prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
        Ec = L.CostVolumeEnergy(imL, None, vol, None, prm, D - 1)
        # the labeling of a device run
        S = PMSweep(Ec)
        S.begin()
        S.init(seeded_labels(S, 99))
        S.iteration(0, 1)
        run_lab = Ec.pm_get()[1]
        S.close()
        fields = {"device_run": run_lab, "random_per_pixel": LC.random_plane_field(H, W, 0.0, D - 1.0, 5, beyond=0.05)}
        En = L.NaiveStereoEnergy(imL, imR, L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4), D - 1)
        for kind, E in (("cost_volume", Ec), ("naive", En)):
            for fname, lab in fields.items():
                E.pm_begin(0, labeling=lab)
                ms = timed(lambda: E.pm_init_from_labeling(0), E.stream, reps=3 if quick else 5)
                print(json.dumps(dict(what="pm_init_from_labeling", energy=kind, field=fname, W=W, H=H, D=D, windR=windR, ms=round(ms, 3),
                                      ns_per_px=round(ms * 1e6 / (H * W), 2), gpu=gpu, power_limit=power)), flush=True)
            # the best existing route: 1x1-target calls of a plan, on a band of rows
            rows = 4 if windR > 20 else 8
            y0 = H // 2
            ys, xs = np.mgrid[y0:y0 + rows, 0:W]
            ys, xs = ys.ravel(), xs.ravel()
            plan = E.make_plan(LC.filter_rects(H, W, windR, ys, xs), np.stack([xs, ys, np.ones_like(xs), np.ones_like(xs)], 1))
            out = torch.zeros((H, W), device="cuda", dtype=torch.float32)
            torch.cuda.synchronize()
            planes = np.ascontiguousarray(fields["random_per_pixel"][ys, xs])
            d_planes = torch.from_numpy(planes).cuda()
            torch.cuda.synchronize()
            ms = timed(lambda: plan.eval_device(d_planes.data_ptr(), out.data_ptr(), W * 4, planes_on_device=True), E.stream,
                       warmup=1, reps=2 if quick else 3)
            print(json.dumps(dict(what="plan_eval_device_1x1", energy=kind, W=W, H=H, D=D, windR=windR, pixels=len(ys), ms=round(ms, 3),
                                  ns_per_px=round(ms * 1e6 / len(ys), 2), gpu=gpu, power_limit=power)), flush=True)
            plan.close()
        # the compiled reference's own branch on a crop
        if LC.reference_available():
            vol_host = vol.cpu().numpy()
            scene = (imL, imR, vol_host, vol_host)
            from oracle import ref_binding as R
            lab = fields["random_per_pixel"]
            for kind in ("cost_volume", "naive"):
                naive = kind == "naive"
                ref = (R.RefEnergy(imL, imR, windR=windR, eps=1e-4, th_col=10.0, th_grad=2.0, alpha=0.9, max_disp=D - 1.0, kind=1) if naive
                       else R.RefEnergy(imL, imR, vol_host, vol_host, windR=windR, eps=1e-4, th_col=0.5, max_disp=D - 1.0, kind=0))
                cy, cx = np.mgrid[H // 2:H // 2 + 16, W // 2:W // 2 + 64]
                units = np.stack([cx.ravel(), cy.ravel(), np.ones(cx.size, int), np.ones(cx.size, int)], 1).astype(np.int32)
                cost = np.zeros((H, W), np.float32)
                cl = np.zeros((H, W, 4), np.float32)
                t = time.perf_counter()
                ref.pm_init(units, lab[cy.ravel(), cx.ravel()], windR, cost, cl, nthreads=16)
                dt = time.perf_counter() - t
                print(json.dumps(dict(what="reference_ref_pm_init_1x1", energy=kind, W=W, H=H, D=D, windR=windR, pixels=int(cx.size),
                                      host_threads=16, ms=round(dt * 1e3, 3), ns_per_px=round(dt * 1e9 / cx.size, 1))), flush=True)
                ref.close()
            del scene, vol_host
        Ec.close()
        En.close()
        del vol
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
