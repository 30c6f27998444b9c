"""Time per launch and per tile of the narrow wgmma convolutions (the 16/32/64-column tiles, which run two CTAs per SM), per
config-4 launch shape.

One eager joint step (D step on MR + CT, G step on CT, B = 8 per domain, dropout keep 0.75) is run once with every wgmma
launch recorded.  Each distinct geometry of a forward that fuses its batch-norm sums and of a data gradient whose tile has
at most 64 columns is then timed on its own through `pnp_conv2d_tc_fwd` / `pnp_conv2d_tc_dgrad` on fresh random operand
planes, dropout and accumulate as in the step: CUDA events around `--launches` back-to-back launches after a warm-up,
median of `--rounds` rounds.

`--lib PATH` (repeatable) times other builds of libpnp_b200.so in the same process, alternating with each other every
round, so that two builds can be compared under the same clocks.  The package's own library is always the first.

Prints the card name and its power limit with the numbers, one JSON line at the end.

    python scripts/bench_conv_tiles.py [--lib other/libpnp_b200.so] [--launches 200] [--rounds 3] [--batch 8]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_conv_epilogue import _power_limit  # noqa: E402


def _block_n(c):
    return 128 if c % 128 == 0 else (64 if c % 64 == 0 else (32 if c % 32 == 0 else 16))


def _tiles(g, fwd, n_cols, ksplit):
    """tiles the persistent CTAs walk (conv_tc.cu run_tc): 128-pixel tiles of every phase x n-tiles x split-K factor; a
    data gradient of stride s is s * s phase convolutions, each over its own output sub-grid"""
    s = 1 if fwd else g.stride
    H, W = (g.Ho, g.Wo) if fwd else (g.H, g.W)
    phases = [((H - py + s - 1) // s, (W - px + s - 1) // s) for py in range(s) for px in range(s)]
    U, V = max(p[0] for p in phases), max(p[1] for p in phases)
    if V >= 128:
        tw, th, tn = 128, 1, 1
    else:
        tw, th = V, min(128 // V, U)
        tn = min(max(128 // (tw * th), 1) if th == U else 1, g.B)
    m = sum(-(-Vp // tw) * -(-Up // th) for Up, Vp in phases) * -(-g.B // tn)
    return m * ((g.Cout if fwd else g.Cin) // n_cols) * ksplit


def _record_launches(B, keep_prob):
    """-> {(kind, geometry tuple, nterms, dropout on / accumulate): launches per joint step} of the narrow-tile launches"""
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
        key = None
        if name == "pnp_conv2d_tc_fwd" and args[9] is not None:
            g = args[5]._obj
            if _block_n(g.Cout) <= 64:
                key = ("fwd+bn", tuple(getattr(g, f) for f, _ in g._fields_), int(args[6]), args[7] is not None)
        elif name == "pnp_conv2d_tc_dgrad":
            g = args[5]._obj
            if _block_n(g.Cin) <= 64:
                key = ("dgrad", tuple(getattr(g, f) for f, _ in g._fields_), int(args[6]), bool(args[7]))
        if key is not None:
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
    for name in ("pnp_conv2d_tc_fwd", "pnp_conv2d_tc_dgrad"):
        getattr(lib, name).argtypes = _C.SIGNATURES[name]
        getattr(lib, name).restype = ctypes.c_int
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
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print("card: %s, power limit: %s; SM-us/tile = us per launch x %d SMs / tiles walked" % (card, plimit, sms))
    shapes = _record_launches(a.batch, a.keep_prob)
    libs = [("this tree", _C.lib)] + [(p, _bind(os.path.abspath(p))) for p in a.lib]
    dev = rt.device()
    seed = torch.tensor([0x5EED], dtype=torch.int64, device=dev)
    gen = torch.Generator(device="cpu").manual_seed(0)
    rows = []
    for (kind, gt, nterms, flag), count in sorted(shapes.items(), key=lambda kv: (kv[0][0], -kv[1] * np.prod(kv[0][1][4:7]))):
        g = _C.ConvGeom(*gt)
        fwd = kind != "dgrad"
        src = (g.B, g.H, g.W, g.Cin) if fwd else (g.B, g.Ho, g.Wo, g.Cout)
        planes = []
        for shape in (src, (g.kh * g.kw * g.Cout * g.Cin,)):
            x = torch.randn(shape, generator=gen).to(dev)
            planes += [x.to(torch.bfloat16), (x - x.to(torch.bfloat16).float()).to(torch.bfloat16)]
        out = torch.zeros((g.B, g.Ho, g.Wo, g.Cout) if fwd else (g.B, g.H, g.W, g.Cin), device=dev)
        stats = torch.zeros(2, g.Cout, dtype=torch.float64, device=dev)
        drop = ctypes.byref(_C.DropCfg(seed.data_ptr(), 7, a.keep_prob)) if fwd and flag else None
        lo_x, lo_w = (planes[1], planes[3]) if nterms == 3 else (None, None)

        def run(lib, n):
            for _ in range(n):
                if fwd:
                    rc = lib.pnp_conv2d_tc_fwd(planes[0].data_ptr(), _C.ptr(lo_x), planes[2].data_ptr(), _C.ptr(lo_w), out.data_ptr(),
                                               ctypes.byref(g), nterms, drop, 0, stats[0].data_ptr(), stats[1].data_ptr(), rt.stream())
                else:
                    rc = lib.pnp_conv2d_tc_dgrad(planes[0].data_ptr(), _C.ptr(lo_x), planes[2].data_ptr(), _C.ptr(lo_w), out.data_ptr(),
                                                 ctypes.byref(g), nterms, int(flag), rt.stream())
                if rc != 0:
                    raise RuntimeError("%s failed: %d" % (kind, rc))

        us = {li: [] for li in range(len(libs))}
        for _ in range(a.rounds):
            for li, (_, lib) in enumerate(libs):
                run(lib, a.warmup)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(lib, a.launches)
                e1.record()
                torch.cuda.synchronize()
                us[li].append(e0.elapsed_time(e1) * 1e3 / a.launches)
        run(_C.lib, 1)
        torch.cuda.synchronize()
        n_, k_, s_ = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
        _C.lib.pnp_tc_last_config(ctypes.byref(n_), ctypes.byref(k_), ctypes.byref(s_))
        ctas, grid = ctypes.c_int(0), ctypes.c_int(0)
        _C.lib.pnp_tc_last_residency(ctypes.byref(ctas), ctypes.byref(grid))
        Ho, Wo = (g.Ho, g.Wo) if fwd else (g.H, g.W)
        tiles = _tiles(g, fwd, n_.value, s_.value)
        row = {"kind": kind, "geom": "B%d %dx%d %d->%d k%d s%d d%d" % (g.B, g.H, g.W, g.Cin, g.Cout, g.kh, g.stride, g.dil),
               "out": "%dx%d" % (Ho, Wo), "kernel": "<%d,%d,%d>%s" % (n_.value, nterms, k_.value, " ksplit %d" % s_.value if s_.value > 1 else ""),
               "ctas_per_sm": ctas.value, "grid": grid.value, "flag": flag, "per_step": count, "tiles": tiles,
               "us": [round(float(np.median(us[li])), 2) for li in range(len(libs))]}
        rows.append(row)
        print("%-6s %-30s out %-8s %-18s %s x%-2d %d/SM grid %3d | " % (kind, row["geom"], row["out"], row["kernel"],
                                                                    ("drop" if fwd else "acc") + str(int(flag)), count, ctas.value, grid.value)
              + " | ".join("%8.1f us %6.2f SM-us/tile" % (u, u * sms / tiles) for u in row["us"]), flush=True)
        del planes, out, stats
    totals = [round(sum(r["us"][li] * r["per_step"] for r in rows) / 1e3, 3) for li in range(len(libs))]
    for (name, _), t in zip(libs, totals):
        print("%s: these launches take %.3f ms per config-4 step" % (name, t))
    print(json.dumps({"card": card, "power_limit": plimit, "batch": a.batch, "launches": a.launches, "rounds": a.rounds,
                      "libs": [n for n, _ in libs], "ms_per_step": totals, "shapes": rows}))


if __name__ == "__main__":
    main()
