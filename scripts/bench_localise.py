"""Cost of the heart localisation (localise.py) on a seeded 512 x 512 x 300 phantom CT scan of 0.7 x 0.7 x 0.5 mm (a 358 mm field
of view) whose heart sits off-centre in a larger body (the structures of bench_volume_source.py, shifted to centre at 40 / 58 / 55 % of
the axes: a 140 x 161 x 80 mm whole-heart box, 60 seed windows), C = 5, with the GAN trainer at B = 8:
* one pnp_native_accumulate launch, one pnp_native_accumulated_labels launch and one pnp_label_boxes call on the native grid,
  timed with CUDA events (best of several rounds of several launches);
* one subject end to end (native.segment's steps): scan load, the seed pass, each iteration, the final prediction, and host I/O
  (the NIfTI write), each with a host clock around work that ends in a device synchronise; one measurement after the
  prediction's shapes were warmed up.  The network holds seeded weights, so where it "finds" the heart says nothing about a
  trained network: only the cost is measured.
Prints the card name and its power limit with the numbers, one JSON line at the end."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_volume_source import STRUCTURES, _power_limit  # noqa: E402


def phantom(directory, shape=(512, 512, 300), spacing=(0.7, 0.7, 0.5), seed=0, size=1.0):
    """the CT-like subject of bench_volume_source.phantom with its heart at `size`, off-centre -> (image path, label path)"""
    from pnp_b200 import nifti
    rng = np.random.RandomState(seed)
    g = np.ogrid[:shape[0], :shape[1], :shape[2]]
    lab = np.zeros(shape, np.int16)
    shift = np.array([0.40, 0.58, 0.55]) - 0.5 * size
    for v, centre, radii in STRUCTURES:
        c, r = (np.array(centre) * size + shift) * shape, np.array(radii) * size * shape
        lab[(((g[0] - c[0]) / r[0]) ** 2 + ((g[1] - c[1]) / r[1]) ** 2 + ((g[2] - c[2]) / r[2]) ** 2) <= 1.0] = v
    body = (((g[0] - shape[0] / 2.0) / (0.48 * shape[0])) ** 2 + ((g[1] - shape[1] / 2.0) / (0.45 * shape[1])) ** 2) <= 1.0
    img = (rng.standard_normal(shape).astype(np.float32) * 40.0 - 900.0 + body * 850.0 + (lab > 0) * 300.0).astype(np.int16)
    aff = np.diag(list(spacing) + [1.0])
    ip, lp = os.path.join(directory, "ct_train_1001_image.nii.gz"), os.path.join(directory, "ct_train_1001_label.nii.gz")
    nifti.save(img, aff, ip)
    nifti.save(lab, aff, lp)
    return ip, lp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=10, help="launches per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="rounds")
    ap.add_argument("--batch-size", type=int, default=8)
    a = ap.parse_args()
    import logging
    import torch
    assert torch.cuda.is_available(), "this benchmark measures the GPU and needs one"
    logging.basicConfig(level=logging.INFO)
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F, localise, native, preprocess, runtime as rt
    card, power = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit %s" % (card, power))
    res = {"card": card, "power_limit": power, "batch_size": a.batch_size}
    tmp = tempfile.mkdtemp(prefix="pnp_bench_localise_")
    image, label = phantom(tmp)
    cal = localise.calibrate([(image, label)])
    rt.set_conv_backend("auto")
    torch.manual_seed(0)
    trainer = native.build_trainer("gan", None, a.batch_size)
    nc = 5
    logits = trainer._ct_logits
    # ---- the kernels, on the ground-truth crop's prediction ------------------------------------------------------------------
    s = preprocess.Subject(image, label)
    scores = native.predict_scores(s, logits, a.batch_size, nc)
    vmap = torch.from_numpy(native.map32(s)).cuda()
    acc = F.NativeAccumulator(s.native_shape, nc)
    gt = native.ground_truth(label)
    out = torch.empty(s.native_shape, dtype=torch.uint8, device="cuda")
    boxes = torch.empty(nc, 7, dtype=torch.int64, device="cuda")
    m0, m1, m2 = s.native_shape
    from pnp_b200._C import call, ptr
    runs = {
        "accumulate": lambda: acc.add(scores, vmap),
        "accumulated_labels": lambda: acc.labels(gt, out),
        "label_boxes": lambda: call("pnp_label_boxes", ptr(out), m0, m1, m2, nc, ptr(boxes), rt.stream()),
    }
    for fn in runs.values():
        fn()
    times = {k: [] for k in runs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.rounds):
        for k, fn in runs.items():
            e0.record()
            for _ in range(a.launches):
                fn()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) / a.launches)
    res["sums_MB"] = acc.sums.numel() * 4 / 1e6
    res["kernel_ms"] = {k: min(v) for k, v in times.items()}
    res["kernel_ms_spread"] = {k: [min(v), max(v)] for k, v in times.items()}
    for k, v in times.items():
        print("%s: %.3f ms (best of %d rounds of %d launches; spread %.3f .. %.3f ms)" % (k, min(v), a.rounds, a.launches, min(v),
                                                                                            max(v)))
    del acc, scores, out
    torch.cuda.empty_cache()

    # ---- one subject end to end ----------------------------------------------------------------------------------------------
    def clock(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return r, time.perf_counter() - t

    t = {"iterations": []}
    scan, t["scan_load"] = clock(lambda: preprocess.Scan(image))
    predict = lambda subj: native.predict_scores(subj, logits, a.batch_size, nc)
    marks = []
    base_locate = localise.locate

    def timed_predict(subj):
        r = predict(subj)
        torch.cuda.synchronize()
        marks.append(time.perf_counter())
        return r

    windows = localise.seed_windows(scan.raw.shape, scan.spacing, cal)
    start = time.perf_counter()
    found, total = clock(lambda: base_locate(scan, timed_predict, cal, nc))
    seed_end = marks[len(marks) - found.iterations - 1] if found.iterations else marks[-1]
    t["seed_s"] = seed_end - start
    prev = seed_end
    for mk in marks[len(marks) - found.iterations:] if found.iterations else []:
        t["iterations"].append(mk - prev)
        prev = mk
    t["locate_total_s"] = total
    res["windows"], res["windows_planned"], res["iterations"], res["converged"] = found.windows, len(windows), found.iterations, \
        found.converged
    if found.subject is not None:
        r, t["final_prediction_and_write"] = clock(lambda: native.evaluate_subject(logits, found.subject, None, tmp, a.batch_size, nc))
        _, t["nifti_write"] = clock(lambda: native.write_prediction(found.subject, np.zeros(scan.native_shape, np.uint8), tmp, nc))
        res["located_box"] = found.subject.box
    res["subject_s"] = t
    print("seed windows %d (%d planned), iterations %d, converged %s, boxes %s" % (found.windows, len(windows), found.iterations,
                                                                                   found.converged, found.boxes))
    print("subject end to end: " + ", ".join("%s %s" % (k, ("%.3f s" % v) if not isinstance(v, list) else
                                                         "[%s] s" % ", ".join("%.3f" % x for x in v)) for k, v in t.items()))
    res.update(native_shape=list(scan.native_shape), truth_box=s.box)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
