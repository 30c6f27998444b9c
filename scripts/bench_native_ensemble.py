"""Cost of native-grid ensembles on the seeded 512 x 512 x 300 phantom CT subject of bench_native_eval.py (D = 261 prepared frames,
C = 5), with the GAN trainer at B = 8:
* pnp_native_labels_ensemble at K = 1, 2, 4, 8 and 16 members with distinct test-time maps (rotations and scales within the
  training ranges), against pnp_native_labels, in alternating rounds timed with CUDA events;
* one subject end to end at K = 1 and at K = 8 (2 checkpoints x 4 rotations), split into native.evaluate_subject's steps (loading,
  prediction with the checkpoint swaps, ground-truth load, resampling, surface distances, NIfTI write, and for the ensemble the
  snapshot and restore of the variables), each with a host clock around work that ends in a device synchronise; one
  measurement each, after the prediction's shapes were warmed up.
Prints the card name and its power limit with the numbers, one JSON line at the end."""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_volume_source import _power_limit, phantom  # noqa: E402

MEMBERS = (1, 2, 4, 8, 16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=10, help="launches per timed window")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds")
    ap.add_argument("--batch-size", type=int, default=8)
    a = ap.parse_args()
    import numpy as np
    import torch
    assert torch.cuda.is_available(), "this benchmark measures the GPU and needs one"
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F, native, preprocess, runtime as rt
    card, power = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit %s" % (card, power))
    res = {"card": card, "power_limit": power, "batch_size": a.batch_size}
    tmp = tempfile.mkdtemp(prefix="pnp_bench_ensemble_")
    image, label = phantom(tmp)
    rt.set_conv_backend("auto")
    torch.manual_seed(0)
    trainer = native.build_trainer("gan", None, a.batch_size)
    nc = 5
    s = preprocess.Subject(image, label)
    gt = native.ground_truth(label)
    one = native.predict_scores(s, trainer._ct_logits, a.batch_size, nc)
    # ---- the resampling launch: K members, every one a copy of the prediction seen through its own test-time map -------------
    tta = [(r, sc, sc, 0.0, 0.0) for sc in (1.0, 0.95) for r in (0.0, -12.0, -8.0, -4.0, 4.0, 8.0, 12.0, 15.0)]
    maps = torch.from_numpy(np.stack([native.member_map32(s, T) for T in native.tta_transforms(tta)])).cuda()
    buf = torch.empty((max(MEMBERS),) + tuple(one.shape), dtype=torch.float32, device="cuda")
    buf.copy_(one.expand_as(buf))
    del one
    out = torch.empty(s.native_shape, dtype=torch.uint8, device="cuda")
    single = lambda: F.native_labels(buf[0], maps[0], s.native_shape, gt, out)
    runs = {"single": single}
    for K in MEMBERS:
        runs[K] = (lambda K=K: F.native_labels(buf[:K], maps[:K], s.native_shape, gt, out))
    lab1, cm1 = F.native_labels(buf[:1], maps[:1], s.native_shape, gt)
    lab0, cm0 = single()
    res["k1_equals_single"] = bool(torch.equal(lab0, lab1) and torch.equal(cm0, cm1))
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
    res["native_labels_ms"] = min(times["single"])
    res["ensemble_ms"] = {str(K): min(times[K]) for K in MEMBERS}
    print("pnp_native_labels: %.3f ms (best of %d rounds of %d launches; %d native voxels, C = %d, with counts)" % (
        res["native_labels_ms"], a.rounds, a.launches, out.numel(), nc))
    for K in MEMBERS:
        print("pnp_native_labels_ensemble K = %2d: %.3f ms (%.2f x the single launch), spread over rounds %.3f .. %.3f ms" % (
            K, min(times[K]), min(times[K]) / res["native_labels_ms"], min(times[K]), max(times[K])))
    print("K = 1 labels and counts equal pnp_native_labels': %s" % res["k1_equals_single"])
    del buf
    torch.cuda.empty_cache()
    # ---- one subject end to end: K = 1 and 2 checkpoints x 4 rotations ------------------------------------------------------------
    ck = []
    state = rt.state_dict()
    for i, scale in enumerate((1.0, 0.98)):
        path = os.path.join(tmp, "ck%d.npz" % i)
        np.savez(path, **{k: (v * np.float32(scale)).astype(v.dtype) if v.dtype == np.float32 else v for k, v in state.items()})
        ck.append(path)
    ens = native.Ensemble(trainer.net, ck, native.tta_transforms([(r, 1.0, 1.0, 0.0, 0.0) for r in (-10.0, -3.0, 3.0, 10.0)]),
                          native.SLOT_KEYWORDS + ("cls",), strip_suffix=True)
    res["workspace_MB_per_member"] = native.workspace_bytes(s, 1, nc) / 1e6

    def clock(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return out, time.perf_counter() - t

    def labels_of(scores, maps, gt_dev, subj):
        if maps is None:
            labels, _ = native.native_prediction(subj, scores, gt_dev)
        else:
            labels, _ = F.native_labels(scores, maps, subj.native_shape, gt_dev)
            F.native_labels(scores[0], maps[0], subj.native_shape, gt_dev)          # dice_first
        return labels.cpu().numpy()

    def phases(e):
        """native.evaluate_subject's steps, each on the clock; their sum is the subject end to end"""
        t = {}
        subj, t["load"] = clock(lambda: preprocess.Subject(image, label))
        if e is None:
            scores, t["prediction"] = clock(lambda: native.predict_scores(subj, trainer._ct_logits, a.batch_size, nc))
            maps = None
        else:
            ctx = e.preserved()
            _, t["state_snapshot"] = clock(ctx.__enter__)
            (scores, maps), t["prediction"] = clock(
                lambda: native.ensemble_scores(subj, trainer._ct_logits, a.batch_size, nc, e))   # with the checkpoint swaps
        gt_dev, t["ground_truth_load"] = clock(lambda: native.ground_truth(label))
        labels, t["resampling"] = clock(lambda: labels_of(scores, maps, gt_dev, subj))
        del scores
        gt_host = gt_dev.cpu().numpy()
        _, t["surface_distances"] = clock(lambda: native.surface_mm(subj, labels, gt_host, nc))
        _, t["nifti_write"] = clock(lambda: native.write_prediction(subj, labels, tmp, nc))
        if e is not None:
            _, t["state_restore"] = clock(lambda: ctx.__exit__(None, None, None))
        t["total"] = sum(t.values())
        return t

    for key, e in (("subject_k1_s", None), ("subject_k8_s", ens)):
        res[key] = phases(e)
        print("subject %s, K = %d: %s" % (s.name, 1 if e is None else e.K,
                                          ", ".join("%s %.3f s" % (k, v) for k, v in res[key].items())))
    print("score buffer %.0f MB per member" % res["workspace_MB_per_member"])
    res.update(native_shape=list(s.native_shape), prepared_frames=s.D)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
