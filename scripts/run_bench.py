"""Wall time of every phase of a whole run (FastGCStereo::run on the device, DESIGN.md 3h): initialisation (random start), each pm iteration,
each graph-cut iteration, the two-view post-processing, and the evaluations -- on the MiddV2 cones pair (tests/golden/middv2_cones) and on
a synthetic 2048x1536x256 cost-volume pair.  The run is issued phase by phase through the same calls lexp_run makes (with the seeds of
sweep.run_seed) and the stream is synchronised after each phase.  Not a gate; prints one JSON line per scene.

--debug-images adds the reference's debug images (DESIGN.md 3j) at every point where lexp_run_ex renders them: per point, the wall time
of rendering and reading back D, N and E of one view (lexp_render_evaluation) or both C images (lexp_render_consistency), and of writing
them as PNG files (cli.imwrite, into a temporary directory).  These times are outside the phases' times, as they are outside a run's timer.

    python scripts/run_bench.py [--scene cones|synthetic|both] [--pm 2] [--iterations 5] [--synthetic-iterations 1] [--dual 1]
                                [--debug-images]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402

import localexpstereo_b200 as L   # noqa: E402
from localexpstereo_b200 import cli   # noqa: E402
from localexpstereo_b200.sweep import RUN_GC, RUN_INIT, RUN_PM, V3_PROPOSERS_REFERENCE, NativePMSweep, run_seed, v3_layer_units   # noqa: E402


def timed_run(E, views, pm, gc, units, props, seed, precision, threshold, debug_images=False):
    t = {"init": 0.0, "pm": [], "gc": [], "post": 0.0, "evaluate": 0.0}
    if debug_images:
        t["images"] = []   # {"index", "images": "D N E of view m" / "C", "render_readback", "png_write"}
    acc = {}
    sw = {m: NativePMSweep(E, unit_sizes=units, proposers=props, mode=m) for m in views}
    tmp = tempfile.TemporaryDirectory() if debug_images else None
    index = [0]

    def write(images, names):
        t0 = time.perf_counter()
        for im, name in zip(images, names):
            cli.imwrite(os.path.join(tmp.name, name), im)
        return time.perf_counter() - t0

    def ev(m):
        t0 = time.perf_counter()
        acc[m] = E.evaluate(m, precision, threshold)
        t["evaluate"] += time.perf_counter() - t0
        if debug_images:
            t0 = time.perf_counter()
            images = E.render_evaluation(m, precision, threshold)
            dt = time.perf_counter() - t0
            png = write(images, ["result%d%s%02d.png" % (m, k, index[0]) for k in "DNE"])
            t["images"].append({"index": index[0], "images": "D N E of view %d" % m, "render_readback": dt, "png_write": png})

    def check_images():
        if debug_images and len(views) == 2:
            t0 = time.perf_counter()
            images = E.render_consistency()
            dt = time.perf_counter() - t0
            png = write(images, ["result%dC%02d.png" % (m, index[0]) for m in (0, 1)])
            t["images"].append({"index": index[0], "images": "C", "render_readback": dt, "png_write": png})
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
                index[0] += 1
                for m in views:
                    ev(m)
                check_images()
        if len(views) == 2:
            t0 = time.perf_counter()
            E.post_process(1.5)
            t["post"] = time.perf_counter() - t0
            index[0] += 1
            for m in views:
                ev(m)
            check_images()
    finally:
        for s in sw.values():
            s.close()
        if tmp is not None:
            tmp.cleanup()
    t["total_without_evaluate"] = t["init"] + sum(t["pm"]) + sum(t["gc"]) + t["post"]
    return t, acc[0]


def cones(args):
    o = cli.parse_args(["-mode", "MiddV2", "-targetDir", os.path.join(ROOT, "tests", "golden", "middv2_cones")])
    E, units, props, precision, threshold = cli.make_energy(o, cli.load_data(o["targetDir"] + "/"))
    try:
        views = (0, 1) if args.dual else (0,)
        t, acc = timed_run(E, views, args.pm, args.iterations, units, props, args.seed, precision, threshold, args.debug_images)
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
        t, _ = timed_run(E, views, args.pm, args.synthetic_iterations, v3_layer_units(W), V3_PROPOSERS_REFERENCE, args.seed, -1.0, 1.0,
                         args.debug_images)
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
    ap.add_argument("--debug-images", action="store_true", help="also time rendering and writing the reference's debug images")
    args = ap.parse_args()
    import torch
    gpu = torch.cuda.get_device_name(0)
    try:   # a read-only query: the power limit is part of every number measured here
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        gpu += ", power limit " + q.stdout.strip() if q.returncode == 0 else ""
    except (OSError, subprocess.TimeoutExpired):
        pass
    for name, fn in (("cones", cones), ("synthetic", synthetic)):
        if args.scene in (name, "both"):
            r = fn(args)
            r["gpu"] = gpu
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
