"""Cost of the per-organ surface distances (ASSD / HD, `functional.surface_distances`) on the GPU it runs on, next to scipy.

For each synthetic subject -- seeded, 256 x 256 x D label volumes (D = 256 and a ragged depth), four ellipsoid organs in the
ground truth and a shifted, resized, speckled copy as the prediction, five classes -- it reports
* the pnp_surface_distance launch sequence alone: CUDA events around `--calls` back-to-back calls after warm-up, per call;
* `surface_distances` end to end (upload of both volumes, the call, the copy back; host clock, median of `--calls`);
* the scipy.ndimage form of oracle/surface_exact.py on the same subject on the host cores (one process per organ), and the
  largest relative difference between the two results.

Prints the card name and its power limit with the numbers, one JSON line at the end.

    python scripts/bench_surface_distance.py [--calls 20] [--depths 256,131] [--no-scipy]
"""
import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NUM_CLS = 5


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=20)
        return out.stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def subject(depth, seed):
    """(pred, gt) uint8 [256, 256, depth]"""
    rng = np.random.default_rng(seed)
    shape = (256, 256, depth)
    g = np.ogrid[:shape[0], :shape[1], :shape[2]]
    gt, pred = np.zeros(shape, np.uint8), np.zeros(shape, np.uint8)
    for c in range(1, NUM_CLS):
        centre = rng.uniform(0.3, 0.7, 3) * shape
        radii = rng.uniform(0.12, 0.3, 3) * shape
        gt[sum(((g[a] - centre[a]) / radii[a]) ** 2 for a in range(3)) < 1] = c
        centre_p = centre + rng.normal(0, 3, 3)
        radii_p = radii * rng.uniform(0.9, 1.1, 3)
        pred[sum(((g[a] - centre_p[a]) / radii_p[a]) ** 2 for a in range(3)) < 1] = c
    speckle = rng.random(shape) < 2e-4
    pred[speckle] = rng.integers(0, NUM_CLS, int(speckle.sum()))
    return pred, gt


def _scipy_class(args):
    from oracle.surface_exact import scipy_raw
    pred, gt, c = args
    return scipy_raw((pred == c).astype(np.uint8), (gt == c).astype(np.uint8), 2)[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--depths", default="256,131")
    ap.add_argument("--no-scipy", action="store_true")
    a = ap.parse_args()
    import ctypes
    import torch
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C, functional as F, runtime as rt
    card, plimit = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit: %s, host cores: %d" % (card, plimit, os.cpu_count()))
    dev = rt.device()
    results = []
    for depth in [int(x) for x in a.depths.split(",")]:
        pred, gt = subject(depth, depth)
        n0, n1, n2 = pred.shape
        nbytes = ctypes.c_longlong(0)
        _C.call("pnp_surface_distance_workspace", n0, n1, n2, NUM_CLS, ctypes.byref(nbytes))
        dp, dg = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        out = torch.empty((NUM_CLS - 1) * 6, dtype=torch.float64, device=dev)
        args = (dp.data_ptr(), dg.data_ptr(), n0, n1, n2, NUM_CLS, None, ws.data_ptr(), nbytes.value, out.data_ptr(), rt.stream())
        for _ in range(3):
            _C.call("pnp_surface_distance", *args)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.calls):
            _C.call("pnp_surface_distance", *args)
        e1.record()
        torch.cuda.synchronize()
        kernel_ms = e0.elapsed_time(e1) / a.calls
        e2e_ms = {}
        for dtype in (np.uint8, np.int16):         # uint8 goes up as it is; wider labels (the test protocol's int16) are mapped first
            p_in, g_in = pred.astype(dtype), gt.astype(dtype)
            F.surface_distances(p_in, g_in, NUM_CLS)
            times = []
            for _ in range(a.calls):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                got = F.surface_distances(p_in, g_in, NUM_CLS)
                times.append(time.perf_counter() - t0)
            e2e_ms[np.dtype(dtype).name] = round(float(np.median(times)) * 1e3, 3)
        row = {"shape": [n0, n1, n2], "workspace_mb": round(nbytes.value / 2 ** 20, 1), "kernel_ms": round(kernel_ms, 3),
               "end_to_end_ms": e2e_ms, "assd": [round(float(x), 4) for x in got["assd"][1:]],
               "hd": [round(float(x), 4) for x in got["hd"][1:]], "border_gt": [int(x) for x in got["border_gt"][1:]]}
        print("%d x %d x %d, 4 organs: pnp_surface_distance %.3f ms per call (%d calls), surface_distances end to end (median) "
              "%.3f ms from uint8 / %.3f ms from int16 volumes, workspace %.1f MiB"
              % (n0, n1, n2, kernel_ms, a.calls, e2e_ms["uint8"], e2e_ms["int16"], row["workspace_mb"]))
        if not a.no_scipy:
            from oracle.surface_exact import metrics
            t0 = time.perf_counter()
            with mp.get_context("fork").Pool(NUM_CLS - 1) as pool:
                ref = np.array(pool.map(_scipy_class, [(pred, gt, c) for c in range(1, NUM_CLS)]))
            scipy_s = time.perf_counter() - t0
            ref = metrics(ref)
            rel = max(float(np.max(np.abs(got[k][1:] - ref[k][1:]) / np.abs(ref[k][1:]))) for k in ("assd", "hd"))
            same_counts = bool(np.array_equal(got["border_pred"], ref["border_pred"]) and np.array_equal(got["border_gt"], ref["border_gt"]))
            row.update(scipy_s=round(scipy_s, 2), scipy_processes=NUM_CLS - 1, max_rel_diff_vs_scipy=rel, border_counts_equal=same_counts)
            print("  scipy.ndimage (%d processes): %.2f s; max relative difference of ASSD / HD vs the GPU: %.3g; border counts "
                  "equal: %s" % (NUM_CLS - 1, scipy_s, rel, same_counts))
        results.append(row)
        del dp, dg, ws, out
    print(json.dumps({"card": card, "power_limit": plimit, "subjects": results}))


if __name__ == "__main__":
    main()
