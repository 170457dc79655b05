"""Time lexp_post_process (PMStereoBase::postProcess on the device) at 2048 x 1536, windR 20, with about 5 %, 15 % and 30 % failed pixels,
next to the reference's own postProcess compiled in oracle/_ref/liblexp_ref_post.so (when present) on the host's cores.

Device: CUDA events on the context's stream around the call (five launches; the weight table upload is included), median of --reps
after --warmup calls, each from the same uploaded snapshot.  Reference: wall time of one call with OpenMP on --threads threads
(default: all cores).  Prints one JSON line per scene."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=1536)
    ap.add_argument("--width", type=int, default=2048)
    ap.add_argument("--windR", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--no-ref", action="store_true")
    a = ap.parse_args()
    import torch
    import test_gpu_post as G
    R = None if a.no_ref else G.ref_lib()
    H, W = a.height, a.width
    for frac in (0.025, 0.08, 0.17):
        im0, im1, lab0, lab1 = G.random_scene(H, W, frac, seed=int(frac * 1000))
        E = G.make_energy(im0, im1, a.windR)
        stream = torch.cuda.ExternalStream(E.stream)
        times = []
        fail = np.zeros((2, H, W), np.uint8)
        for it in range(a.warmup + a.reps):
            E.pm_begin(0, None, lab0)
            E.pm_begin(1, None, lab1)
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(stream)
            E.post_process(1.5, fail if it == 0 else None)
            t1.record(stream)
            t1.synchronize()
            if it >= a.warmup:
                times.append(t0.elapsed_time(t1))
        n_failed = int((fail > 0).sum())
        res = dict(H=H, W=W, windR=a.windR, failed_fraction=round(n_failed / (2 * H * W), 4), failed_pixels=n_failed,
                   device_ms=round(statistics.median(times), 3), device_ms_min=round(min(times), 3), device_ms_max=round(max(times), 3),
                   gpu=torch.cuda.get_device_name(0))
        E.close()
        if R is not None:
            h = R.ref_post_create(H, W, im0.ctypes.data, im1.ctypes.data, a.windR, G.OMEGA, 64.0)
            o0, o1 = lab0.copy(), lab1.copy()
            t = time.perf_counter()
            assert R.ref_post_process(h, o0.ctypes.data, o1.ctypes.data, H, W, 1.5, a.threads) == 0
            res.update(reference_s=round(time.perf_counter() - t, 3), reference_threads=a.threads)
            R.ref_post_destroy(h)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
