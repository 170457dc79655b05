"""Wall time of every phase of a whole run (FastGCStereo::run on the device, DESIGN.md 3h): initialisation (random start), each pm iteration,
each graph-cut iteration, the two-view post-processing, and the evaluations -- on the MiddV2 cones pair (tests/golden/middv2_cones) and on
a synthetic 2048x1536x256 cost-volume pair.  The run is issued phase by phase through the same calls lexp_run makes (with the seeds of
sweep.run_seed) and the stream is synchronised after each phase.  Not a gate; prints one JSON line per scene.

    python scripts/run_bench.py [--scene cones|synthetic|both] [--pm 2] [--iterations 5] [--synthetic-iterations 1] [--dual 1]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402

import localexpstereo_b200 as L   # noqa: E402
from localexpstereo_b200 import cli   # noqa: E402
from localexpstereo_b200.sweep import RUN_GC, RUN_INIT, RUN_PM, V3_PROPOSERS_REFERENCE, NativePMSweep, run_seed, v3_layer_units   # noqa: E402


def timed_run(E, views, pm, gc, units, props, seed, precision, threshold):
    t = {"init": 0.0, "pm": [], "gc": [], "post": 0.0, "evaluate": 0.0}
    acc = {}
    sw = {m: NativePMSweep(E, unit_sizes=units, proposers=props, mode=m) for m in views}

    def ev(m):
        t0 = time.perf_counter()
        acc[m] = E.evaluate(m, precision, threshold)
        t["evaluate"] += time.perf_counter() - t0
    try:
        t0 = time.perf_counter()
        for m in views:
            sw[m].begin()
            sw[m].random_start(run_seed(seed, m, RUN_INIT))
        E.sync()
        t["init"] = time.perf_counter() - t0
        for m in views:
            ev(m)
        for phase, n, key in ((RUN_PM, pm, "pm"), (RUN_GC, gc, "gc")):
            for it in range(n):
                t0 = time.perf_counter()
                for m in views:
                    (sw[m].iteration if phase == RUN_PM else sw[m].gc_iteration)(it, run_seed(seed, m, phase, it))
                E.sync()
                t[key].append(time.perf_counter() - t0)
                for m in views:
                    ev(m)
        if len(views) == 2:
            t0 = time.perf_counter()
            E.post_process(1.5)
            t["post"] = time.perf_counter() - t0
            for m in views:
                ev(m)
    finally:
        for s in sw.values():
            s.close()
    t["total_without_evaluate"] = t["init"] + sum(t["pm"]) + sum(t["gc"]) + t["post"]
    return t, acc[0]


def cones(args):
    o = cli.parse_args(["-mode", "MiddV2", "-targetDir", os.path.join(ROOT, "tests", "golden", "middv2_cones")])
    E, units, props, precision, threshold = cli.make_energy(o, cli.load_data(o["targetDir"] + "/"))
    try:
        views = (0, 1) if args.dual else (0,)
        t, acc = timed_run(E, views, args.pm, args.iterations, units, props, args.seed, precision, threshold)
    finally:
        E.close()
    return {"scene": "MiddV2 cones 450x375, ndisp 59, image-based energy", "views": len(views), "seconds": t,
            "all": acc["all"], "nonocc": acc["nonocc"]}


def synthetic(args):
    from oracle import lexp_oracle as O
    H, W, D = 1536, 2048, 256
    imL, imR = O.synthetic_image(H, W, 42), O.synthetic_image(H, W, 43)
    volL = O.synthetic_volume(D, H, W, 1234)
    prm = L.Parameters(lambda_=0.5, windR=20, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, imR, volL, None, prm, D - 1)
    try:
        E.set_volume(1, volL, L.VOL_RIGHT_FROM_LEFT)
        del volL
        E.set_smoothness(prm.lambda_, prm.omega, prm.th_smooth, prm.epsilon)
        E.set_ground_truth(np.full((H, W), np.float32(D / 2)), None)
        views = (0, 1) if args.dual else (0,)
        t, _ = timed_run(E, views, args.pm, args.synthetic_iterations, v3_layer_units(W), V3_PROPOSERS_REFERENCE, args.seed, -1.0, 1.0)
    finally:
        E.close()
    return {"scene": "synthetic 2048x1536x256, cost-volume energy", "views": len(views), "seconds": t}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", default="both", choices=["cones", "synthetic", "both"])
    ap.add_argument("--pm", type=int, default=2)
    ap.add_argument("--iterations", type=int, default=5)
    ap.add_argument("--synthetic-iterations", type=int, default=1)
    ap.add_argument("--dual", type=int, default=1)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    import torch
    gpu = torch.cuda.get_device_name(0)
    for name, fn in (("cones", cones), ("synthetic", synthetic)):
        if args.scene in (name, "both"):
            r = fn(args)
            r["gpu"] = gpu
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
