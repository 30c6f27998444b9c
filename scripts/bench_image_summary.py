"""Cost of the opt-in image summaries (`--image-summaries`) on the GPU it runs on:

* the pnp_image_summary_u8 kernel for the GAN trainer's six panel sources at B = 8 (3 images each, 18 panels of 256 x 256):
  CUDA events around `--launches` back-to-back launches, reported per launch;
* the wall time of one GAN `output_minibatch_stats` monitoring pass at B = 8 with and without image summaries (median of
  `--passes`; with images it includes the one device->host copy, the PNG encoding on the host and the event write).

Prints the card name and its power limit with the numbers, one JSON line at the end.

    python scripts/bench_image_summary.py [--launches 200] [--passes 15] [--batch 8]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=20)
        return out.stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--passes", type=int, default=15)
    ap.add_argument("--batch", type=int, default=8)
    a = ap.parse_args()
    import torch
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C, adversarial as adv, functional as F, runtime as rt
    from pnp_b200.train_gan import configure
    card, plimit = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit: %s" % (card, plimit))
    B, dev = a.batch, rt.device()
    g = torch.Generator(device="cpu").manual_seed(0)
    ct, mr = (torch.randn(B, 256, 256, 3, generator=g).to(dev) for _ in range(2))
    lab = [torch.randint(0, 5, (B, 256, 256), generator=g).to(dev) for _ in range(2)]
    cty, mry = (F.one_hot(l, 5) for l in lab)
    lct, lmr = (torch.randn(B, 256, 256, 5, generator=g).to(dev) for _ in range(2))

    # ---- the kernel alone -------------------------------------------------------------------------------------------------
    srcs = [(lct, 2, 0), (ct, 0, 1), (cty, 1, 0), (lmr, 2, 0), (mr, 0, 1), (mry, 1, 0)]
    n = min(B, 3)
    out = torch.empty(len(srcs), n, 256, 256, dtype=torch.uint8, device=dev)
    ia = lambda v: (ctypes.c_int * len(srcs))(*v)
    args = ((ctypes.c_void_p * len(srcs))(*[t.data_ptr() for t, _, _ in srcs]), ia([k for _, k, _ in srcs]),
            ia([t.shape[3] for t, _, _ in srcs]), ia([c for _, _, c in srcs]), len(srcs), B, 256, 256, n, out.data_ptr(), rt.stream())
    for _ in range(20):
        _C.call("pnp_image_summary_u8", *args)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.launches):
        _C.call("pnp_image_summary_u8", *args)
    e1.record()
    torch.cuda.synchronize()
    kernel_us = e0.elapsed_time(e1) * 1e3 / a.launches
    print("pnp_image_summary_u8, 6 sources x %d images at B = %d: %.1f us per launch (%d launches)" % (n, B, kernel_us, a.launches))

    # ---- one GAN monitoring pass with and without images -----------------------------------------------------------------------
    ck, nc, tc = configure("train-gan")
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
    tr = adv.Trainer(net, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc)
    log = tempfile.mkdtemp(prefix="pnp_imgbench_")
    res = {}
    for label, on in (("scalars", False), ("scalars+images", True), ("scalars#2", False), ("scalars+images#2", True)):
        times = []
        for i in range(a.passes + 3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.output_minibatch_stats(i, ct, cty, mr, mry, log_dir=os.path.join(log, label), image_summaries=on)
            torch.cuda.synchronize()
            if i >= 3:
                times.append(time.perf_counter() - t0)
        res.setdefault(label.split("#")[0], []).append(float(np.median(times)) * 1e3)
    for k, v in res.items():
        print("output_minibatch_stats (%s), median of %d passes, two alternating rounds: %s ms" % (k, a.passes, " / ".join("%.1f" % x for x in v)))
    print(json.dumps({"card": card, "power_limit": plimit, "batch": B, "kernel_us": round(kernel_us, 2),
                      "pass_ms_scalars": [round(x, 2) for x in res["scalars"]],
                      "pass_ms_scalars_images": [round(x, 2) for x in res["scalars+images"]]}))


if __name__ == "__main__":
    main()
