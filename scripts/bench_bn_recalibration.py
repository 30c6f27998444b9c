"""Cost of batch-norm recalibration (bnstats.py, elementwise.cu pnp_bn_accumulate / pnp_bn_population) on the card it runs on, in
one run:
* `pnp_bn_accumulate` and `pnp_bn_population` alone at the segmenter's table (30 layers, 8 032 channels) and the DAM's (20 layers,
  2 912 channels);
* one recalibration pass (batch-statistics batch norm on the covered layers, keep_prob 1, plus its accumulate launch) against one
  inference forward (moving statistics) at B = 8 and 16, for the segmenter and the GAN trainer's CT stream ('dam'), in
  alternating rounds;
* recalibrate_bn.py end to end (build, restore, --volumes source on the seeded 512 x 512 x 300 phantom of
  bench_volume_source.py, `--batches` passes, write) for the GAN trainer at B = 8.
Times are CUDA events (host clock around a synchronised run for the tool), medians over `--reps` rounds.  Prints the card name and
its power limit with the numbers, one JSON line at the end.

    python scripts/bench_bn_recalibration.py [--launches 200] [--passes 10] [--reps 7] [--batches 200]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_ema import _events  # noqa: E402
from bench_volume_source import _power_limit, phantom  # noqa: E402


def _kernel_cost(moving, launches, reps):
    import torch
    from pnp_b200 import runtime as rt
    from pnp_b200._C import BnAccEntry, BnPopEntry, call, ptr
    n = len(moving)
    sums = [torch.randn(2 * mm.numel(), dtype=torch.float64, device="cuda") for mm, _ in moving]
    acc = [torch.zeros(2 * mm.numel(), dtype=torch.float64, device="cuda") for mm, _ in moving]
    mm_out = [torch.empty_like(mm) for mm, _ in moving]
    mv_out = [torch.empty_like(mv) for _, mv in moving]
    at = (BnAccEntry * n)(*[BnAccEntry(ptr(s), ptr(s) + 8 * mm.numel(), ptr(a), mm.numel()) for s, a, (mm, _) in zip(sums, acc, moving)])
    pt = (BnPopEntry * n)(*[BnPopEntry(ptr(a), 1 << 20, ptr(o), ptr(v), mm.numel()) for a, o, v, (mm, _) in zip(acc, mm_out, mv_out, moving)])
    acc_once = lambda: call("pnp_bn_accumulate", at, n, rt.stream())
    pop_once = lambda: call("pnp_bn_population", pt, n, rt.stream())
    acc_once()
    pop_once()
    a, p = [], []
    for _ in range(reps):
        a.append(_events(acc_once, launches))
        p.append(_events(pop_once, launches))
    return {"layers": n, "channels": sum(mm.numel() for mm, _ in moving), "accumulate_us": 1e3 * statistics.median(a),
            "population_us": 1e3 * statistics.median(p)}


def _pass_cost(kind, B, passes, reps):
    """one recalibration pass (collector active, accumulate launch) against one inference forward, alternating rounds"""
    import torch
    from pnp_b200 import bnstats, native, runtime as rt
    from oracle.pnp_graphs import synthetic_images
    tr = native.build_trainer(kind, None, B)
    x = synthetic_images(B, 7, 0.3, 0.8).cuda()
    if kind == "gan":
        moving = bnstats.covered_statistics([v for v in rt.global_variables() if v.pnp_kind == "bn_moving" and v.pnp_name.startswith("adapt_")])
        recal = lambda: tr.net.segment(x, "ct", 1.0, front_bn=True, joint_bn=False)
        infer = lambda: tr._ct_logits(x)
    else:
        moving = bnstats.covered_statistics([v for v in rt.global_variables() if v.pnp_kind == "bn_moving"])
        recal = lambda: tr.net.forward(x, 1.0, main_bn=True, adapt_bn=True)
        infer = lambda: tr._logits(x)
    r_ms, i_ms = [], []
    with torch.no_grad(), bnstats.collecting(moving) as col:
        def one_pass():
            rt.scratch.begin_step()
            col.begin_pass()
            recal()
            col.end_pass()
        for _ in range(2):
            one_pass()
            infer()
        for _ in range(reps):
            r_ms.append(_events(one_pass, passes))
            i_ms.append(_events(infer, passes))
    r, i = statistics.median(r_ms), statistics.median(i_ms)
    return {"recal_pass_ms": r, "inference_ms": i, "ratio": r / i}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--passes", type=int, default=10)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--batches", type=int, default=200, help="passes of the end-to-end tool run")
    a = ap.parse_args()
    import numpy as np
    import torch
    import pnp_b200  # noqa: F401
    from pnp_b200 import bnstats, lib, native, runtime as rt
    card, power = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit %s" % (card, power))
    res = {"card": card, "power_limit": power}

    for kind, key in (("segmenter", "segmenter_table"), ("gan", "dam_table")):
        native.build_trainer(kind, None, 8)
        mv = [v for v in rt.global_variables() if v.pnp_kind == "bn_moving" and (kind == "segmenter" or v.pnp_name.startswith("adapt_"))]
        res[key] = _kernel_cost(bnstats.covered_statistics(mv), a.launches, a.reps)
        print(key, json.dumps(res[key]))
    for kind in ("segmenter", "gan"):
        for B in (8, 16):
            k = "%s_pass_B%d" % (kind, B)
            res[k] = _pass_cost(kind, B, a.passes, a.reps)
            print(k, json.dumps(res[k]))

    with tempfile.TemporaryDirectory() as tmp:
        image, label = phantom(tmp)
        pairs = os.path.join(tmp, "pairs")
        with open(pairs, "w") as f:
            f.write("%s %s\n" % (image, label))
        native.build_trainer("gan", None, 8)
        st = rt.state_dict()
        st["pnp/global_step"] = np.int64(0)
        ck = lib._save(st, os.path.join(tmp, "latest"))
        torch.cuda.synchronize()
        t0 = time.time()
        bnstats.main(["--trainer", "gan", "--checkpoint", ck, "--out", os.path.join(tmp, "latest_bn.npz"), "--volumes", pairs,
                      "--batches", str(a.batches), "--batch-size", "8"])
        torch.cuda.synchronize()
        res["tool_gan_B8_s"] = time.time() - t0
        res["tool_batches"] = a.batches
        print("tool end to end (gan, B = 8, %d passes, 512 x 512 x 300 phantom): %.2f s" % (a.batches, res["tool_gan_B8_s"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
