"""Cost of drawing augmented training slices on the GPU (`data.VolumeSource`, `pnp_resample_planes`) on the card it runs on.

One seeded phantom CT subject of the MMWHS size -- 512 x 512 x 300 voxels of 0.35 x 0.35 x 0.5 mm, ellipsoid structures carrying
all seven MMWHS values -- is written as .nii.gz to a temporary directory.  The script reports
* the preparation end to end: `prepare_data.prepare` of the subject for the test split (load, crop, z-score, upload, one launch,
  NIfTI write) and for `--records` augmented training records (host clock);
* the pnp_resample_planes launch alone at B = 8 and 16 (3 channels, middle label plane): CUDA events around `--launches` launches
  after warm-up, per launch;
* `VolumeSource.next()` (matrices drawn on the host, one launch; host clock around each call and a device synchronise, median)
  against `TFRecordSource.next()` over the written records plus the host-to-device copy of the batch, at the same B.

Prints the card name and its power limit with the numbers, one JSON line at the end.

    python scripts/bench_volume_source.py [--launches 200] [--calls 50] [--records 64]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STRUCTURES = [(550, (0.45, 0.62, 0.50), (0.10, 0.08, 0.16)), (600, (0.38, 0.45, 0.66), (0.08, 0.07, 0.10)),
              (205, (0.58, 0.48, 0.46), (0.11, 0.10, 0.17)), (500, (0.58, 0.48, 0.46), (0.07, 0.06, 0.11)),
              (420, (0.60, 0.30, 0.62), (0.07, 0.05, 0.09)), (820, (0.50, 0.42, 0.72), (0.035, 0.035, 0.10)),
              (850, (0.42, 0.58, 0.74), (0.035, 0.035, 0.07))]


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=20)
        return out.stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def phantom(directory, shape=(512, 512, 300), spacing=(0.35, 0.35, 0.5), seed=0):
    """a CT-like subject in RAS voxel order as {ct_train_1001_image, _label}.nii.gz -> (image path, label path)"""
    from pnp_b200 import nifti
    rng = np.random.RandomState(seed)
    g = np.ogrid[:shape[0], :shape[1], :shape[2]]
    lab = np.zeros(shape, np.int16)
    for v, centre, radii in STRUCTURES:
        c, r = np.array(centre) * shape, np.array(radii) * shape
        lab[(((g[0] - c[0]) / r[0]) ** 2 + ((g[1] - c[1]) / r[1]) ** 2 + ((g[2] - c[2]) / r[2]) ** 2) <= 1.0] = v
    img = (rng.standard_normal(shape).astype(np.float32) * 40.0 - 50.0 + (lab > 0) * 300.0).astype(np.int16)
    aff = np.diag(list(spacing) + [1.0])
    ip, lp = os.path.join(directory, "ct_train_1001_image.nii.gz"), os.path.join(directory, "ct_train_1001_label.nii.gz")
    nifti.save(img, aff, ip)
    nifti.save(lab, aff, lp)
    return ip, lp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--records", type=int, default=64)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark measures the GPU and needs one"
    import pnp_b200  # noqa: F401
    from pnp_b200 import prepare_data, runtime as rt
    from pnp_b200.data import VolumeSource
    from pnp_b200.functional import resample_planes
    from pnp_b200.tfrecord import TFRecordSource
    card, power = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit %s" % (card, power))
    res = {"card": card, "power_limit": power}
    tmp = tempfile.mkdtemp(prefix="pnp_bench_volume_")
    pair = phantom(tmp)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    prepare_data.prepare("ct", [pair], "test", os.path.join(tmp, "out"))
    torch.cuda.synchronize()
    res["prepare_test_subject_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    lists = prepare_data.prepare("ct", [pair], "train", os.path.join(tmp, "out"), slices_per_volume=a.records, seed=1)
    torch.cuda.synchronize()
    res["prepare_train_records_s"] = time.perf_counter() - t0
    res["prepare_train_records"] = a.records
    print("preparation of one 512 x 512 x 300 subject: test split %.2f s, %d training records %.2f s" % (
        res["prepare_test_subject_s"], a.records, res["prepare_train_records_s"]))
    files = [ln.strip() for ln in open(lists[0]) if ln.strip()]

    for B in (8, 16):
        vs = VolumeSource([pair], B, 1234)
        mats = torch.from_numpy(vs.draw_matrices()).cuda()
        img = torch.empty(B, 256, 256, 3, device="cuda")
        lab = torch.empty(B, 256, 256, dtype=torch.int64, device="cuda")
        for _ in range(10):
            resample_planes(vs.vol, vs.cls, mats, 256, 256, True, 1, img, lab)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.launches):
            resample_planes(vs.vol, vs.cls, mats, 256, 256, True, 1, img, lab)
        e1.record()
        e1.synchronize()
        k_us = e0.elapsed_time(e1) * 1e3 / a.launches
        # bytes the launch must move at least: the outputs (fp32 image + int64 label) -- the gathers hit L2 mostly
        out_bytes = B * 256 * 256 * (3 * 4 + 8)

        def timed(fn, n):
            ts = []
            for _ in range(n):
                torch.cuda.synchronize()
                t = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t)
            return float(np.median(ts)) * 1e3

        for _ in range(5):
            vs.next()
        v_ms = timed(vs.next, a.calls)
        src = TFRecordSource(files, B, seed=1234, num_threads=4)
        dev = rt.device()

        def record_batch():
            x, y = src.next()
            x.to(dev, non_blocking=True)
            y.to(dev, non_blocking=True)

        for _ in range(5):
            record_batch()
        t_ms = timed(record_batch, a.calls)
        src.close()
        print("B = %2d: pnp_resample_planes %.1f us per launch (%.0f GB/s of output); VolumeSource.next() %.3f ms; "
              "TFRecordSource.next() + H2D copy %.3f ms" % (B, k_us, out_bytes / k_us * 1e-3, v_ms, t_ms))
        res["B%d" % B] = {"kernel_us": k_us, "output_GBps": out_bytes / k_us * 1e-3, "volume_source_next_ms": v_ms,
                          "tfrecord_next_plus_h2d_ms": t_ms}
        del vs
    shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
