"""The reference's command line (main.cpp): `python -m localexpstereo_b200 -mode MiddV2|MiddV3 -targetDir D -outputDir O [options]`.

Arguments follow ArgsParser (ArgsParser.h): `-name value` pairs, booleans as true / false / an integer; Options (main.cpp:14-51) gives
the defaults, smooth_weight 1.0 for MiddV2 and 0.5 for MiddV3.  `-seed N` is an addition: the reference seeds cv::theRNG() from time(NULL)
(main.cpp:430-450); here the run seed defaults to 0, so a command repeats its result.  `-threadNum` is accepted and ignored.

Outputs as the reference's: disp0.pfm, disp0raw.pfm (-doDual only), time.txt, debug/log_output.txt (the Evaluator's log of view 0),
the Evaluator's images debug/result{m}D{ii}.png, result{m}N{ii}.png and result{m}E{ii}.png of every view at every evaluation
(Evaluator.h:164-166), with -doDual the consistency-check images debug/result0C{ii}.png / result1C{ii}.png after every iteration and the
post-processing (FastGCStereo.h:160-167,188-195,208-215), and one console line per evaluation of view 0 (Evaluator.h:183).  The whole
run is one lexp_run_ex call on the device, which renders the images there."""
from __future__ import annotations

import os
import sys

import numpy as np

OPTION_TYPES = {"mode": str, "outputDir": str, "targetDir": str, "threadNum": int, "doDual": bool, "iterations": int, "pmIterations": int,
                "ndisp": int, "filterRadious": int, "smooth_weight": float, "mc_threshold": float, "seed": int}


def _convert(kind, s):   # ArgsParser::convertStringToValue
    if kind is bool:
        return True if s == "true" else False if s == "false" else _stoi(s) != 0
    if kind is int:
        return _stoi(s)
    if kind is float:
        return float(s)
    return s


def _stoi(s):
    """std::stoi: leading whitespace, an optional sign and the longest run of digits."""
    t = s.lstrip()
    i = 1 if t[:1] in "+-" else 0
    while i < len(t) and t[i].isdigit():
        i += 1
    if i == 0 or not t[:i].lstrip("+-"):
        raise ValueError(f"not an integer: {s!r}")
    return int(t[:i])


def parse_args(argv):
    """ArgsParser + Options::loadOptionValues (main.cpp:31-51): a dict of every option."""
    amap = {}
    i = 0
    while i < len(argv):
        if argv[i].startswith("-") and i + 1 < len(argv):
            amap[argv[i][1:]] = argv[i + 1]
            i += 2
        else:
            i += 1
    o = dict(mode="", outputDir="", targetDir="", iterations=5, pmIterations=2, doDual=False, ndisp=0, smooth_weight=1.0,
             mc_threshold=0.5, filterRadious=20, threadNum=-1, seed=0)
    for k in ("outputDir", "targetDir", "mode"):
        if k in amap:
            o[k] = amap[k]
    if o["mode"] == "MiddV2":
        o["smooth_weight"] = 1.0
    elif o["mode"] == "MiddV3":
        o["smooth_weight"] = 0.5
    for k in ("threadNum", "doDual", "iterations", "pmIterations", "ndisp", "filterRadious", "smooth_weight", "mc_threshold", "seed"):
        if k in amap:
            o[k] = _convert(OPTION_TYPES[k], amap[k])
    return o


def imread(path, gray=False):
    """cv::imread (BGR, or IMREAD_GRAYSCALE): cv2 where it is importable, else PIL.  None if the file does not exist."""
    if not os.path.exists(path):
        return None
    try:
        import cv2
        im = cv2.imread(path, cv2.IMREAD_GRAYSCALE if gray else cv2.IMREAD_COLOR)
        if im is not None:
            return im
    except ImportError:
        pass
    from PIL import Image
    with Image.open(path) as im:
        if gray:
            return np.array(im.convert("L"))
        return np.ascontiguousarray(np.array(im.convert("RGB"))[..., ::-1])


def imwrite(path, image):
    """cv::imwrite of an 8-bit image, gray [H][W] or BGR [H][W][3]: cv2 where it is importable, else PIL.  Raises if the file cannot be
    written."""
    try:
        import cv2
    except ImportError:
        cv2 = None
    if cv2 is not None:
        if not cv2.imwrite(path, image):
            raise OSError(f"could not write {path}")
        return
    from PIL import Image
    Image.fromarray(np.ascontiguousarray(image[..., ::-1] if image.ndim == 3 else image)).save(path)


def read_pfm(path):
    """cvutils::io::read_pfm_file for a one-channel file: rows stored bottom-up, little-endian when the scale is negative."""
    if not os.path.exists(path):
        return None
    with open(path, "rb") as f:
        if f.readline().strip() != b"Pf":
            raise ValueError(f"{path}: not a one-channel pfm file")
        w, h = (int(t) for t in f.readline().split())
        scale = float(f.readline())
        a = np.frombuffer(f.read(4 * w * h), dtype="<f4" if scale < 0 else ">f4").reshape(h, w)
    return np.ascontiguousarray(a[::-1].astype(np.float32))


def read_calib(path):
    """Calib(calib.txt) (main.cpp:76-140): the `key=value` lines; ndisp is what the run needs."""
    c = {"ndisp": 0, "gt_prec": -1.0}
    if os.path.exists(path):
        for line in open(path):
            if "=" in line:
                k, v = (t.strip() for t in line.split("=", 1))
                if k == "ndisp":
                    c["ndisp"] = _stoi(v)
    return c


def load_data(d, ndisp=0):
    """loadData (main.cpp:201-268): (imL, imR, dispGT, nonocc, ndisp, gt_prec), or None when the pair or ndisp is missing."""
    gt_prec = -1.0
    info = os.path.join(d, "info.txt")
    if os.path.exists(info):
        vals = open(info).read().split()
        gt_scale = int(vals[0])
        gt_prec = float(np.float32(1.0) / np.float32(gt_scale))
        if ndisp <= 0 and len(vals) > 1:
            ndisp = int(vals[1])
    else:
        c = read_calib(os.path.join(d, "calib.txt"))
        gt_prec = c["gt_prec"]
        if ndisp <= 0:
            ndisp = c["ndisp"]
    if ndisp <= 0:
        print("ndisp is not speficied.")
        return None
    im0, im1 = imread(os.path.join(d, "imL.png")), imread(os.path.join(d, "imR.png"))
    if im0 is None or im1 is None:
        im0, im1 = imread(os.path.join(d, "im0.png")), imread(os.path.join(d, "im1.png"))
        if im0 is None or im1 is None:
            print(f"Image pairs (im0.png, im1.png) or (imL.png, imR.png) not found in\n{d}")
            return None
    g = imread(os.path.join(d, "groundtruth.png"), gray=True)
    if g is not None:
        gt = g.astype(np.float32)
        if gt_prec > 0:   # convertTo(CV_32F, gt_prec): double product rounded to float
            gt = (g.astype(np.float64) * np.float64(np.float32(gt_prec))).astype(np.float32)
        gt[g == 0] = np.inf
    else:
        gt = read_pfm(os.path.join(d, "disp0GT.pfm"))
    if gt is None:
        gt = np.zeros(im0.shape[:2], np.float32)
    nonocc = imread(os.path.join(d, "nonocc.png"), gray=True)
    if nonocc is None:
        nonocc = imread(os.path.join(d, "mask0nocc.png"), gray=True)
    nonocc = np.where(nonocc == 255, 255, 0).astype(np.uint8) if nonocc is not None else np.full(im0.shape[:2], 255, np.uint8)
    return im0, im1, gt, nonocc, ndisp, gt_prec


def disparities(labeling):
    """computeDisparities (StereoEnergy.h:269-272) of a Plane [H][W] labeling on the host: a x + b y + c + v 0, rounded to float at every
    step, as the device computes it (lexp_get_disparities)."""
    H, W = labeling.shape[:2]
    x = np.arange(W, dtype=np.float32)[None, :]
    y = np.arange(H, dtype=np.float32)[:, None]
    with np.errstate(invalid="ignore", over="ignore"):
        return np.ascontiguousarray(((labeling[..., 0] * x + labeling[..., 1] * y) + labeling[..., 2]) + labeling[..., 3] * np.float32(0.0))


def error_threshold_v3(target_dir):   # main.cpp:342-346
    if "trainingQ" in target_dir or "testQ" in target_dir:
        return 0.5
    if "trainingF" in target_dir or "testF" in target_dir:
        return 2.0
    return 1.0


def make_energy(o, data):
    """The energy and the run arguments of MidV2 / MidV3 (main.cpp:270-330 / 331-418)."""
    import localexpstereo_b200 as L
    from .sweep import V3_PROPOSERS_REFERENCE, v3_layer_units
    imL, imR, gt, nonocc, ndisp, gt_prec = data
    maxdisp = float(ndisp - 1)
    if o["mode"] == "MiddV2":
        prm = L.Parameters(lambda_=o["smooth_weight"], windR=o["filterRadious"], filterName="GF", filter_param1=1e-4)
        E = L.NaiveStereoEnergy(imL, imR, prm, maxdisp)
        units, precision, threshold = [5, 15, 25], gt_prec, 0.5
    else:
        prm = L.Parameters(lambda_=o["smooth_weight"], windR=o["filterRadious"], filterName="GF", filter_param1=1e-4, th_col=o["mc_threshold"])
        E = L.CostVolumeEnergy(imL, imR, None, None, prm, maxdisp)
        d = o["targetDir"]
        E.set_volume_file(0, os.path.join(d, "im0.acrt"), L.VOL_FILL)
        if os.path.exists(os.path.join(d, "im1.acrt")):
            E.set_volume_file(1, os.path.join(d, "im1.acrt"), L.VOL_FILL)
        else:
            print("Cost volume file im1.acrt not found so recovered from im0.acrt.")
            E.set_volume_file(1, os.path.join(d, "im0.acrt"), L.VOL_RIGHT_FROM_LEFT)
        units, precision, threshold = v3_layer_units(imL.shape[1]), -1.0, error_threshold_v3(d)
    E.set_smoothness(prm.lambda_, prm.omega, prm.th_smooth, prm.epsilon)
    E.set_ground_truth(gt, nonocc)
    return E, units, V3_PROPOSERS_REFERENCE, precision, threshold


def run(o, out=sys.stdout):
    """MidV2 / MidV3 with the options `o` (parse_args): writes the reference's output files.  Returns the list of view-0 log rows."""
    if o["mode"] not in ("MiddV2", "MiddV3"):
        raise SystemExit("-mode must be MiddV2 or MiddV3")
    out.write(f"Running by Middlebury {'V2' if o['mode'] == 'MiddV2' else 'V3'} mode.\n")
    data = load_data(os.path.join(o["targetDir"], ""), o["ndisp"])   # -ndisp wins over info.txt / calib.txt in both modes
    if data is None:
        return None
    if o["mode"] == "MiddV3" and not os.path.exists(os.path.join(o["targetDir"], "im0.acrt")):
        out.write("Cost volume file im0.acrt not found\n")
        return None
    outdir = o["outputDir"]
    os.makedirs(os.path.join(outdir, "debug"), exist_ok=True)
    E, units, props, precision, threshold = make_energy(o, data)
    rows = []
    try:
        with open(os.path.join(outdir, "debug", "log_output.txt"), "w") as log:
            log.write("Time\tEng\tData\tSmooth\tall\tnonocc\n")
            log.flush()

            def cb(index, mode, r, seconds):
                if mode != 0:
                    return
                row = (seconds, r["energy"], r["data"], r["smooth"], r["all"], r["nonocc"])
                rows.append(row)
                log.write("%f\t%f\t%f\t%f\t%f\t%f\n" % row)
                log.flush()
                out.write("%2d %5.1f\t%.0f\t%.0f\t%.0f\t%4.2f\t%4.2f\n" % ((index,) + row))
            def image_cb(index, mode, kind, image):   # Evaluator.h:164-166 (header "result"), FastGCStereo.h:164-165
                imwrite(os.path.join(outdir, "debug", "result%d%s%02d.png" % (mode, kind, index)), image)
            views = (0, 1) if o["doDual"] else (0,)
            lab, raw = E.run(o["iterations"], views, o["pmIterations"], None, units, props, o["seed"], precision, threshold, callback=cb,
                             image_callback=image_cb)
        from .energy import save_pfm_file
        save_pfm_file(os.path.join(outdir, "disp0.pfm"), disparities(lab))
        if o["doDual"]:
            save_pfm_file(os.path.join(outdir, "disp0raw.pfm"), disparities(raw))
        with open(os.path.join(outdir, "time.txt"), "w") as f:
            f.write("%f\n" % (rows[-1][0] if rows else 0.0))
    finally:
        E.close()
    return rows


def main(argv=None):
    o = parse_args(sys.argv[1:] if argv is None else argv)
    for k in ("mode", "outputDir", "targetDir", "iterations", "pmIterations", "doDual", "ndisp", "filterRadious", "smooth_weight",
              "mc_threshold", "seed"):
        print(f"{k}\t{o[k]}")
    rows = run(o)
    return 0 if rows is not None else 1
