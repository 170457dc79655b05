"""Cost of the device RansacProposer (LEXP_PROP_RANSAC) at 2048 x 1536 x 256, windR 20, measured with CUDA events:
  * one pm iteration and one graph-cut iteration with sweep.V3_PROPOSERS_REFERENCE against sweep.V3_PROPOSERS_DEVICE (the same
    number of evaluations per cell, the RANSAC slot given to one more RandomProposer draw),
  * the RANSAC launches alone, per layer, from the state after init and after one pm iteration (the inlier ratios, and with them
    the number of samples each cell draws, differ a lot between the two).
Prints one JSON line; run on an H100 (it refuses to run without a GPU)."""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import GCSweep, V3_PROPOSERS_DEVICE, V3_PROPOSERS_REFERENCE, pm_seed
    assert torch.cuda.is_available(), "needs a GPU"
    W, H, D, windR = 2048, 1536, 256, 20
    imL = synth.synthetic_image(H, W, 42)
    vol = np.random.default_rng(1234).random((D, H, W), dtype=np.float32)
    E = L.CostVolumeEnergy(imL, None, vol, None, L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4), D - 1)
    del vol
    ev = lambda: torch.cuda.Event(enable_timing=True)
    stream = torch.cuda.Stream()
    E.set_stream(stream.cuda_stream)

    def timed(fn):
        a, b = ev(), ev()
        torch.cuda.synchronize()
        a.record(stream)
        fn()
        b.record(stream)
        torch.cuda.synchronize()
        return a.elapsed_time(b)

    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                            capture_output=True, text=True).stdout.strip()
    except OSError:
        out["power_limit"] = "unknown"
    sweeps = {name: GCSweep(E, proposers=props) for name, props in (("device", V3_PROPOSERS_DEVICE), ("reference", V3_PROPOSERS_REFERENCE))}
    labels = synth.synthetic_planes(sweeps["device"].init_units, 1, D, 7)[0]
    E.set_smoothness()
    REPS = 3
    for name in ("device", "reference"):
        S = sweeps[name]
        pm, gc = [], []
        for r in range(REPS + 1):   # the first round warms every shape up
            S.begin(); S.init(labels)
            t_pm = timed(lambda: S.iteration(0, 5))
            t_gc = timed(lambda: S.gc_iteration(1, 5))
            if r:
                pm.append(t_pm); gc.append(t_gc)
        out[f"pm_iteration_ms_{name}"] = [round(t, 1) for t in pm]
        out[f"gc_iteration_ms_{name}"] = [round(t, 1) for t in gc]
    # the RANSAC launches alone: one pm_step of kind RANSAC per group of a layer (the fused launch that evaluates the proposals is
    # included: it is part of the step); minus the same steps with ExpansionProposer, which costs one fused launch and no fit
    S = sweeps["reference"]
    for when in ("init", "iteration"):
        S.begin(); S.init(labels)
        if when == "iteration":
            S.iteration(0, 5)
        torch.cuda.synchronize()
        cost, lab = S.get()
        for li in range(3):
            groups = [g for (l, gi, g, _) in S.schedule if l == li and g is not None]
            res = {}
            for kind, kname in ((L.PROP_RANSAC, "ransac"), (L.PROP_EXPANSION, "expansion")):
                ts = []
                for r in range(REPS + 1):
                    E.pm_begin(0, cost, lab)
                    E.pm_reset_sync()
                    t = timed(lambda: [g.plan.pm_step(0, kind, 0, pm_seed(5, 0, 0, li, g.group, 1)) for g in groups])
                    if r:
                        ts.append(t)
                res[kname] = round(float(np.median(ts)), 2)
            out[f"layer{li}_after_{when}_ms"] = res
    print(json.dumps(out))
    for S in sweeps.values():
        S.close()
    E.close()


if __name__ == "__main__":
    main()
