"""Cost of segmenting a subject on its own MMWHS grid (`native.py`, `pnp_native_labels`) on the card it runs on.

One seeded phantom CT subject of the MMWHS size -- 512 x 512 x 300 voxels of 0.35 x 0.35 x 0.5 mm, the structures of
bench_volume_source.py -- is written as .nii.gz to a temporary directory.  The script reports
* the pnp_native_labels call alone (5 classes, with the ground truth and its confusion counts): CUDA events around `--launches`
  launches after warm-up, per launch;
* the subject end to end with the GAN trainer's adapted CT stream at B = 8 (seeded initialisation; the time does not depend on
  the weights), split into loading and cropping the subject, prediction of every prepared frame, loading and uploading the native
  ground truth, resampling onto the native grid (the launch and the copy back), surface distances in mm, and the NIfTI write
  (host clock around work that ends in a device synchronise);
* with `--hd-percentile Q`, surface distances in mm with the Q-th percentile HD end to end, and pnp_surface_distance_pct next to
  pnp_surface_distance on the native prediction and ground truth at native spacing (bench_surface_distance.compare_pct: CUDA
  events, `--rounds` alternating rounds of `--calls` calls).

Prints the card name and its power limit with the numbers, one JSON line at the end.

    python scripts/bench_native_eval.py [--launches 200] [--batch-size 8] [--hd-percentile 95 [--calls 5] [--rounds 3]]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_volume_source import _power_limit, phantom  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--batch-size", type=int, default=8)
    ap.add_argument("--hd-percentile", type=float, default=None, metavar="Q", help="also time pnp_surface_distance_pct at Q")
    ap.add_argument("--calls", type=int, default=5, help="calls per round of the --hd-percentile comparison")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of the --hd-percentile comparison")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark measures the GPU and needs one"
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F, native, preprocess, runtime as rt
    card, power = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit %s" % (card, power))
    res = {"card": card, "power_limit": power, "batch_size": a.batch_size}
    tmp = tempfile.mkdtemp(prefix="pnp_bench_native_")
    image, label = phantom(tmp)
    rt.set_conv_backend("auto")
    torch.manual_seed(0)
    trainer = native.build_trainer("gan", None, a.batch_size)
    nc = 5

    def clock(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return out, time.perf_counter() - t

    s, res["subject_load_s"] = clock(lambda: preprocess.Subject(image, label))
    native.predict_scores(s, trainer._ct_logits, a.batch_size, nc)                 # warm-up: every shape of the timed run
    scores, res["prediction_s"] = clock(lambda: native.predict_scores(s, trainer._ct_logits, a.batch_size, nc))

    gt_dev, res["ground_truth_load_s"] = clock(lambda: native.ground_truth(label))

    def resample():
        labels, cm = native.native_prediction(s, scores, gt_dev)
        return labels.cpu().numpy(), cm
    (labels, cm), res["resampling_s"] = clock(resample)
    gt = gt_dev.cpu().numpy()
    _, res["surface_distances_s"] = clock(lambda: native.surface_mm(s, labels, gt, nc))
    _, res["nifti_write_s"] = clock(lambda: native.write_prediction(s, labels, tmp, nc))
    res.update(native_shape=list(s.native_shape), prepared_frames=s.D)
    print("subject %s on %s, D = %d prepared frames: load %.2f s, prediction %.3f s, ground-truth load %.2f s, resampling %.3f s, "
          "surface distances %.3f s, NIfTI write %.2f s" % (s.name, s.native_shape, s.D, res["subject_load_s"], res["prediction_s"],
                                                           res["ground_truth_load_s"], res["resampling_s"], res["surface_distances_s"],
                                                           res["nifti_write_s"]))

    vmap = torch.from_numpy(native.map32(s)).cuda()
    out = torch.empty(s.native_shape, dtype=torch.uint8, device="cuda")
    for _ in range(10):
        F.native_labels(scores, vmap, s.native_shape, gt_dev, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.launches):
        F.native_labels(scores, vmap, s.native_shape, gt_dev, out)
    e1.record()
    e1.synchronize()
    k_ms = e0.elapsed_time(e1) / a.launches
    # bytes the launch must move at least: the labels written and the ground truth read (the score gathers hit L2 mostly)
    voxels = int(out.numel())
    res.update(kernel_ms=k_ms, kernel_launches=a.launches, native_voxels=voxels, kernel_Gvoxel_per_s=voxels / k_ms * 1e-6)
    print("pnp_native_labels: %.3f ms per launch over %d launches, %.1f G native voxels/s (%d voxels, %d classes, with counts)" % (
        k_ms, a.launches, voxels / k_ms * 1e-6, voxels, nc))
    if a.hd_percentile is not None:
        from bench_surface_distance import compare_pct, print_pct
        _, res["surface_distances_pct_s"] = clock(lambda: native.surface_mm(s, labels, gt, nc, a.hd_percentile))
        print("surface distances with hd%g: %.3f s end to end" % (a.hd_percentile, res["surface_distances_pct_s"]))
        res["pct"] = compare_pct(out, gt_dev, nc, a.hd_percentile, a.calls, a.rounds, native.native_spacing(s))
        print_pct(res["pct"])
    shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
