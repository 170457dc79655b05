"""Mints tests/golden/cones_run_ref.json: the reference's own whole-run accuracy on the MiddV2 cones pair (tests/golden/middv2_cones),
`-mode MiddV2 -doDual 1`, 2 pm + 5 graph-cut iterations, error threshold 0.5, for three seeds -- FastGCStereo::run and Evaluator.h
compiled from the reference's sources (oracle/build_ref_run.py).  Run from the repository root where the reference sources are present:
    python tests/golden/make_cones_run_ref.py"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from localexpstereo_b200 import cli   # noqa: E402
from oracle import build_ref_run, ref_run   # noqa: E402

SEEDS = [1, 2, 3]


def main():
    assert build_ref_run.build() is not None, "the reference sources are needed to mint this fixture"
    d = os.path.join(ROOT, "tests", "golden", "middv2_cones") + "/"
    imL, imR, gt, nonocc, ndisp, gt_prec = cli.load_data(d)
    runs = []
    for seed in SEEDS:
        t = time.time()
        r = ref_run.midv2(imL, imR, gt, nonocc, ndisp, gt_prec, seed, iterations=5, pm_iterations=2, do_dual=True)
        runs.append({"seed": seed, "all": r["all"], "nonocc": r["nonocc"], "energy": r["energy"]})
        print(seed, r, "%.0f s" % (time.time() - t), flush=True)
    out = {"config": "MiddV2 cones, -doDual 1, -pmIterations 2, -iterations 5, error threshold 0.5; cv::theRNG() of OpenMP thread j "
                      "seeded with seed + j as main.cpp does", "openmp_threads": os.cpu_count(), "runs": runs}
    with open(os.path.join(ROOT, "tests", "golden", "cones_run_ref.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
