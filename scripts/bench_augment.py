"""Cost of the opt-in elastic and intensity augmentations of `data.VolumeSource` on the card it runs on.

The seeded 512 x 512 x 300 phantom CT subject of scripts/bench_volume_source.py is written to a temporary directory.  At B = 8 and
16 the script times, with CUDA events and medians over `--reps` rounds that alternate the settings within one run:
* the launches alone: the elastic field (pnp_smooth_noise_field, K = 2, sigma 10), the bias field (K = 1, sigma 32) and
  pnp_resample_planes_aug with all fields against plain pnp_resample_planes (3 channels, middle label plane), each over `--launches`
  launches per round;
* `VolumeSource.next()` with the augmentations off, elastic only, and both on (events around one call after a synchronise, so
  the host-side draws are included).
Prints the card name and its power limit with the numbers, one JSON line at the end.

    python scripts/bench_augment.py [--launches 50] [--reps 15]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--reps", type=int, default=15)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark measures the GPU and needs one"
    import pnp_b200  # noqa: F401
    from pnp_b200 import preprocess as pp
    from pnp_b200.data import VolumeSource
    from pnp_b200.functional import resample_planes, smooth_noise_field
    from bench_volume_source import _power_limit, phantom
    card, power = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit %s" % (card, power))
    res = {"card": card, "power_limit": power}
    tmp = tempfile.mkdtemp(prefix="pnp_bench_augment_")
    pair = phantom(tmp)
    S = pp.SIZE

    def events(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e3 / n               # us per call

    for B in (8, 16):
        sources = {"off": VolumeSource([pair], B, 1234), "elastic": VolumeSource([pair], B, 1234, elastic=True),
                   "both": VolumeSource([pair], B, 1234, elastic=True, intensity=True)}
        vs = sources["both"]
        mats = torch.from_numpy(vs.draw_matrices()).cuda()
        img = torch.empty(B, S, S, 3, device="cuda")
        lab = torch.empty(B, S, S, dtype=torch.int64, device="cuda")
        te = torch.from_numpy(pp.gaussian_taps(pp.ELASTIC_SIGMA)).cuda()
        tb = torch.from_numpy(pp.gaussian_taps(pp.BIAS_SIGMA)).cuda()
        disp, gain = torch.empty(B, 2, S, S, device="cuda"), torch.empty(B, 1, S, S, device="cuda")
        scratch = torch.empty(B, 2, S, S, device="cuda")
        ab = torch.tensor([[1.1, 0.05]] * B, device="cuda")
        launches = {
            "elastic_field": lambda: smooth_noise_field(1, 2, B, 2, S, S, te, pp.ELASTIC_ALPHA, -pp.ELASTIC_MAX_PX, pp.ELASTIC_MAX_PX,
                                                        out=disp, tmp=scratch),
            "bias_field": lambda: smooth_noise_field(1, 3, B, 1, S, S, tb, pp.BIAS_BETA, -pp.BIAS_MAX, pp.BIAS_MAX, out=gain,
                                                     tmp=scratch.view(-1)[:B * S * S].view(B, 1, S, S)),
            "resample_plain": lambda: resample_planes(vs.vol, vs.cls, mats, S, S, True, 1, img, lab),
            "resample_aug": lambda: resample_planes(vs.vol, vs.cls, mats, S, S, True, 1, img, lab, disp=disp, gain=gain[:, 0], ab=ab),
        }
        for fn in launches.values():
            for _ in range(5):
                fn()
        for s in sources.values():
            for _ in range(5):
                s.next()
        times = {k: [] for k in list(launches) + ["next_" + k for k in sources]}
        for _ in range(a.reps):
            for k, fn in launches.items():
                times[k].append(events(fn, a.launches))
            for k, s in sources.items():
                times["next_" + k].append(events(s.next, 1))
        med = {k: float(np.median(v)) for k, v in times.items()}
        print("B = %2d: elastic field %.1f us, bias field %.1f us, resample plain %.1f us, resample with all fields %.1f us per "
              "launch; VolumeSource.next() off %.3f ms, elastic %.3f ms, both %.3f ms" % (
                  B, med["elastic_field"], med["bias_field"], med["resample_plain"], med["resample_aug"], med["next_off"] / 1e3,
                  med["next_elastic"] / 1e3, med["next_both"] / 1e3))
        res["B%d" % B] = {k + "_us": v for k, v in med.items()}
        del sources, vs
    shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
