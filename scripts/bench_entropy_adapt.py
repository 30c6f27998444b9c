"""Cost of test-time entropy adaptation (tent.py, elementwise.cu pnp_entropy_*) on the card it runs on, in one run:
* `pnp_entropy_reduce`, `pnp_entropy_finalize` and `pnp_entropy_bwd` alone on C = 5 logits at B = 8 and 16 (256 x 256);
* one adaptation step, eager and captured, for both trainers at B = 8 and 16, against one inference forward and against the
  trainer's own captured training step (the segmenter's Adam step; the GAN trainer's G step at keep_prob 0.75), in alternating
  rounds, and the full-arena Adam launch alone (its share of the captured step);
* adapt_entropy.py end to end (build, restore, --volumes source on the seeded 512 x 512 x 300 phantom of
  bench_volume_source.py, `--steps` steps, `--recalibrate-batches` passes, write) for the GAN trainer at B = 8.
Times are CUDA events (host clock around a synchronised run for the tool), medians over `--reps` rounds.  Prints the card name and
its power limit with the numbers, one JSON line at the end.

    python scripts/bench_entropy_adapt.py [--launches 200] [--steps-per-round 10] [--reps 7] [--tool-steps 100]
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


def _kernel_cost(B, launches, reps):
    import torch
    from pnp_b200 import runtime as rt
    from pnp_b200._C import call, ptr
    C = 5
    P = B * 256 * 256
    x = torch.randn(B, 256, 256, C, device="cuda") * 3.0
    acc = torch.zeros(1 + C, dtype=torch.float64, device="cuda")
    out = torch.empty(1 + C, device="cuda")
    g = torch.ones(1, device="cuda")
    dl = torch.empty_like(x)
    red = lambda: call("pnp_entropy_reduce", ptr(x), P, C, ptr(acc), rt.stream())
    fin = lambda: call("pnp_entropy_finalize", ptr(acc), P, C, ptr(out), rt.stream())
    bwd = lambda: call("pnp_entropy_bwd", ptr(x), ptr(g), ptr(dl), P, C, rt.stream())
    for f in (red, fin, bwd):
        f()
    r, f_, b = [], [], []
    for _ in range(reps):
        r.append(_events(red, launches))
        f_.append(_events(fin, launches))
        b.append(_events(bwd, launches))
    gb = P * C * 4 / 1e9
    res = {"reduce_us": 1e3 * statistics.median(r), "finalize_us": 1e3 * statistics.median(f_), "bwd_us": 1e3 * statistics.median(b)}
    res["reduce_GBps"] = gb / (res["reduce_us"] * 1e-6)
    res["bwd_GBps"] = 2 * gb / (res["bwd_us"] * 1e-6)
    return res


def _step_cost(kind, B, n, reps):
    """one adaptation step eager and replayed, an inference forward, the trainer's captured training step and the Adam launch
    of the adaptation's optimizer, in alternating rounds"""
    import torch
    from pnp_b200 import native
    from oracle.pnp_graphs import synthetic_images
    from tests.models import step_onehot
    tr = native.build_trainer(kind, None, B)
    x = synthetic_images(B, 7, 0.3, 0.8).cuda()
    if kind == "gan":
        infer = lambda: tr._ct_logits(x)
        assert tr.capture_g_step(x, 0.75, warmup=2)
        train = lambda: tr.g_step_replay(x, 0.75)
    else:
        y = step_onehot(B, 9)
        infer = lambda: tr._logits(x)
        assert tr.capture_train_step(x, y, 0.75, warmup=2)
        train = lambda: tr.train_step_replay(x, y, 0.75)
    s = tr.entropy_adaptation(1e-4)
    s.step(x)
    s.step(x)
    captured = s.capture(x)
    eager = lambda: s.step(x)
    replay = lambda: s.replay(x)
    adam = lambda: s.opt.step()
    t = {"eager": [], "captured": [], "inference": [], "train_step": [], "adam": []}
    with torch.no_grad():
        infer()
    for _ in range(reps):
        t["eager"].append(_events(eager, n))
        t["captured"].append(_events(replay, n))
        with torch.no_grad():
            t["inference"].append(_events(infer, n))
        t["train_step"].append(_events(train, n))
        t["adam"].append(_events(adam, n))
    s.restore()
    s.close()
    res = {k + "_ms": statistics.median(v) for k, v in t.items()}
    res["capture_ok"] = bool(captured)
    res["arena_floats"] = s.arena.total
    res["captured_over_inference"] = res["captured_ms"] / res["inference_ms"]
    res["captured_over_train_step"] = res["captured_ms"] / res["train_step_ms"]
    res["adam_share_of_captured"] = res["adam_ms"] / res["captured_ms"]
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps-per-round", type=int, default=10)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--tool-steps", type=int, default=100)
    ap.add_argument("--tool-recalibrate-batches", type=int, default=200)
    a = ap.parse_args()
    import numpy as np
    import torch
    import pnp_b200  # noqa: F401
    from pnp_b200 import lib, native, runtime as rt, tent
    card, power = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit %s" % (card, power))
    res = {"card": card, "power_limit": power}
    for B in (8, 16):
        k = "kernels_B%d" % B
        res[k] = _kernel_cost(B, a.launches, a.reps)
        print(k, json.dumps(res[k]))
    for kind in ("segmenter", "gan"):
        for B in (8, 16):
            k = "%s_step_B%d" % (kind, B)
            res[k] = _step_cost(kind, B, a.steps_per_round, a.reps)
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
        _, hist, _ = tent.main(["--trainer", "gan", "--checkpoint", ck, "--out", os.path.join(tmp, "latest_tent.npz"),
                                "--volumes", pairs, "--steps", str(a.tool_steps), "--recalibrate-batches",
                                str(a.tool_recalibrate_batches), "--batch-size", "8"])
        torch.cuda.synchronize()
        res["tool_gan_B8_s"] = time.time() - t0
        res["tool_steps"], res["tool_recalibrate_batches"] = a.tool_steps, a.tool_recalibrate_batches
        res["tool_entropy_first_last"] = [float(hist[0, 0]), float(hist[-1, 0])]
        print("tool end to end (gan, B = 8, %d steps + %d recalibration passes, 512 x 512 x 300 phantom): %.2f s"
              % (a.tool_steps, a.tool_recalibrate_batches, res["tool_gan_B8_s"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
