"""Cost of the batch-norm partial statistics in the wgmma convolution's epilogue, per layer of one config-4 step.

One eager joint step (D step on MR + CT, G step on CT, B = 8 per domain, dropout keep 0.75) is run once with every
wgmma forward launch recorded.  Each distinct forward geometry that takes its batch-norm sums from the epilogue is then
timed on its own through `pnp_conv2d_tc_fwd`, with the sums on (bn_sum / bn_sumsq set) and off (NULL): CUDA events around
`--launches` back-to-back launches after a warm-up, on fresh random operand planes, dropout as in the step.  The
difference times the number of times the shape runs in one step is the step's cost of the statistics.

`--lib PATH` (repeatable) times other builds of libpnp_b200.so in the same process, alternating with each other every
round, so that two builds can be compared under the same clocks.  The package's own library is always the first.

Prints the card name and its power limit with the numbers, one JSON line at the end.

    python scripts/bench_conv_epilogue.py [--lib other/libpnp_b200.so] [--launches 200] [--rounds 3] [--batch 8]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

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


def _record_bn_launches(B, keep_prob):
    """-> {(geometry tuple, nterms, dropout on): launches per joint step} of the wgmma forwards that fuse BN statistics"""
    import torch
    from pnp_b200 import adversarial as adv, functional as F, runtime as rt
    from pnp_b200.data import SyntheticSource
    from pnp_b200.train_gan import configure
    rt.set_conv_backend("auto")
    torch.manual_seed(0)
    rt.manual_seed(1234)
    ck, nc, tc = configure("train-gan")
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc, stddev=0.05, stddev_plain=0.05)
    tc["dis_sub_iter"] = 1
    tr = adv.Trainer(net, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc)
    dev = rt.device()
    mr = SyntheticSource(B, seed=1234, pool=1).pool[0][0].to(dev)
    ct = SyntheticSource(B, seed=4321, shift=0.3, scale=0.8, pool=1).pool[0][0].to(dev)
    ct2 = SyntheticSource(B, seed=8765, shift=0.3, scale=0.8, pool=1).pool[0][0].to(dev)
    seen = {}
    inner = F._tc_launch

    def spy(tag, flops, name, *args):
        if name == "pnp_conv2d_tc_fwd" and args[9] is not None:
            g = args[5]._obj
            key = (tuple(getattr(g, f) for f, _ in g._fields_), int(args[6]), args[7] is not None)
            seen[key] = seen.get(key, 0) + 1
        return inner(tag, flops, name, *args)

    F._tc_launch = spy
    try:
        tr.d_step(mr, ct, keep_prob)
        tr.g_step(ct2, keep_prob)
        torch.cuda.synchronize()
    finally:
        F._tc_launch = inner
    return seen


def _bind(path):
    from pnp_b200 import _C
    lib = ctypes.CDLL(path)
    lib.pnp_conv2d_tc_fwd.argtypes = _C.SIGNATURES["pnp_conv2d_tc_fwd"]
    lib.pnp_conv2d_tc_fwd.restype = ctypes.c_int
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="another build of libpnp_b200.so to time alongside")
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--keep-prob", type=float, default=0.75)
    a = ap.parse_args()
    import torch
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C, runtime as rt
    card, plimit = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit: %s" % (card, plimit))
    shapes = _record_bn_launches(a.batch, a.keep_prob)
    libs = [("this tree", _C.lib)] + [(p, _bind(os.path.abspath(p))) for p in a.lib]
    dev = rt.device()
    seed = torch.tensor([0x5EED], dtype=torch.int64, device=dev)
    gen = torch.Generator(device="cpu").manual_seed(0)
    rows = []
    for (gt, nterms, drop_on), count in sorted(shapes.items(), key=lambda kv: -kv[1] * np.prod(kv[0][0][4:7])):
        g = _C.ConvGeom(*gt)
        planes = []
        for shape in ((g.B, g.H, g.W, g.Cin), (g.kh * g.kw * g.Cout * g.Cin,)):
            x = torch.randn(shape, generator=gen).to(dev)
            planes += [x.to(torch.bfloat16), (x - x.to(torch.bfloat16).float()).to(torch.bfloat16)]
        y = torch.empty(g.B, g.Ho, g.Wo, g.Cout, device=dev)
        stats = torch.zeros(2, g.Cout, dtype=torch.float64, device=dev)
        drop = ctypes.byref(_C.DropCfg(seed.data_ptr(), 7, a.keep_prob)) if drop_on else None
        lo_x, lo_w = (planes[1], planes[3]) if nterms == 3 else (None, None)

        def run(lib, n, bn):
            for _ in range(n):
                rc = lib.pnp_conv2d_tc_fwd(planes[0].data_ptr(), _C.ptr(lo_x), planes[2].data_ptr(), _C.ptr(lo_w), y.data_ptr(),
                                           ctypes.byref(g), nterms, drop, 0, stats[0].data_ptr() if bn else None,
                                           stats[1].data_ptr() if bn else None, rt.stream())
                if rc != 0:
                    raise RuntimeError("pnp_conv2d_tc_fwd failed: %d" % rc)

        us = {(li, bn): [] for li in range(len(libs)) for bn in (True, False)}
        for _ in range(a.rounds):
            for li, (_, lib) in enumerate(libs):
                for bn in (True, False):
                    run(lib, a.warmup, bn)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    run(lib, a.launches, bn)
                    e1.record()
                    torch.cuda.synchronize()
                    us[(li, bn)].append(e0.elapsed_time(e1) * 1e3 / a.launches)
        n_, k_, s_ = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
        _C.lib.pnp_tc_last_config(ctypes.byref(n_), ctypes.byref(k_), ctypes.byref(s_))
        row = {"geom": "B%d %dx%d %d->%d k%d s%d d%d" % (g.B, g.H, g.W, g.Cin, g.Cout, g.kh, g.stride, g.dil),
               "out": "%dx%d" % (g.Ho, g.Wo), "kernel": "<%d,%d,%d>%s" % (n_.value, nterms, k_.value, " ksplit %d" % s_.value if s_.value > 1 else ""),
               "dropout": drop_on, "per_step": count, "libs": []}
        for li in range(len(libs)):
            on, off = float(np.median(us[(li, True)])), float(np.median(us[(li, False)]))
            row["libs"].append({"bn_on_us": round(on, 2), "bn_off_us": round(off, 2), "gap_us": round(on - off, 2),
                                "gap_ms_per_step": round((on - off) * count / 1e3, 4)})
        rows.append(row)
        print("%-32s out %-8s %-18s drop %d x%-2d | " % (row["geom"], row["out"], row["kernel"], drop_on, count)
              + " | ".join("on %8.1f off %8.1f gap %6.1f us" % (l["bn_on_us"], l["bn_off_us"], l["gap_us"]) for l in row["libs"]),
              flush=True)
        del planes, y, stats
    totals = [round(sum(r["libs"][li]["gap_ms_per_step"] for r in rows), 3) for li in range(len(libs))]
    for (name, _), t in zip(libs, totals):
        print("%s: BN statistics cost %.3f ms per config-4 step (sum over shapes of (on - off) x launches per step)" % (name, t))
    print(json.dumps({"card": card, "power_limit": plimit, "batch": a.batch, "launches": a.launches, "rounds": a.rounds,
                      "libs": [n for n, _ in libs], "ms_per_step": totals, "shapes": rows}))


if __name__ == "__main__":
    main()
