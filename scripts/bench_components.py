"""Cost of keeping the largest connected component of each class (`pnp_largest_components`) on the card it runs on, against
scipy on the host, with a bit-for-bit comparison of the two.

Seeded label volumes, 5 classes:
* the 512 x 512 x 300 native-size phantom of bench_native_eval.py (its four MMWHS structures as class ids), clean and with
  salt-and-pepper islands (0.5 % of the voxels set to a random label 1 .. 6, so out-of-range labels occur too);
* 256^3 voxels of four ellipsoid organs with salt-and-pepper islands at densities 0.1 %, 5 % and 31 % (near the 6-connected
  site-percolation threshold, where components are largest and most tangled).
For each volume and connectivity 6 and 26 it reports the pnp_largest_components call alone (with the clean volume as ground truth
and its confusion counts; CUDA events around `--calls` calls after warm-up, per call), oracle/components_exact.scipy_lcc on the
host (one call, host clock) and whether the two agree bit for bit in the output, the stats and the counts.

Prints the card name and its power limit with the numbers, one JSON line at the end.

    python scripts/bench_components.py [--calls 20]
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_volume_source import STRUCTURES, _power_limit  # noqa: E402
from oracle import components_exact as ce  # noqa: E402

NUM_CLS = 5


def native_phantom():
    """the class ids of bench_native_eval.py's 512 x 512 x 300 phantom subject (bench_volume_source.phantom's labels)"""
    from pnp_b200 import preprocess
    shape = (512, 512, 300)
    g = np.ogrid[:shape[0], :shape[1], :shape[2]]
    lab = np.zeros(shape, np.int16)
    for v, centre, radii in STRUCTURES:
        c, r = np.array(centre) * shape, np.array(radii) * shape
        lab[(((g[0] - c[0]) / r[0]) ** 2 + ((g[1] - c[1]) / r[1]) ** 2 + ((g[2] - c[2]) / r[2]) ** 2) <= 1.0] = v
    return np.ascontiguousarray(preprocess.map_labels(lab)[0], dtype=np.uint8)


def organs(n=256):
    """four ellipsoid organs, classes 1 .. 4, in an n^3 volume"""
    i, j, k = np.ogrid[:n, :n, :n]
    lab = np.zeros((n, n, n), np.uint8)
    for c, (ci, cj, ck, r) in enumerate([(0.5, 0.45, 0.5, 0.2), (0.42, 0.62, 0.38, 0.13), (0.6, 0.38, 0.62, 0.15),
                                         (0.33, 0.5, 0.68, 0.08)], 1):
        lab[((i - ci * n) ** 2 + (j - cj * n) ** 2 + (k - ck * n) ** 2) <= (r * n) ** 2] = c
    return lab


def salt(lab, density, seed):
    rng = np.random.RandomState(seed)
    out = lab.copy()
    hit = rng.rand(*lab.shape) < density
    out[hit] = rng.randint(1, NUM_CLS + 2, size=int(hit.sum()))
    return out


def measure(name, lab, gt, calls):
    import torch
    from pnp_b200 import _C, runtime as rt
    n0, n1, n2 = lab.shape
    dl, dg = torch.from_numpy(lab).cuda(), torch.from_numpy(gt).cuda()
    out = torch.empty_like(dl)
    stats = torch.empty(NUM_CLS, 3, dtype=torch.int64, device="cuda")
    cm = torch.empty(NUM_CLS, NUM_CLS, dtype=torch.int64, device="cuda")
    rows = []
    for conn in (6, 26):
        nb = ctypes.c_longlong(0)
        _C.call("pnp_largest_components_workspace", n0, n1, n2, NUM_CLS, conn, ctypes.byref(nb))
        ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")

        def once():
            _C.call("pnp_largest_components", _C.ptr(dl), n0, n1, n2, NUM_CLS, conn, _C.ptr(out), _C.ptr(dg), _C.ptr(cm),
                    _C.ptr(stats), _C.ptr(ws), nb.value, rt.stream())
        for _ in range(3):
            once()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            once()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1) / calls
        got = (out.cpu().numpy(), stats.cpu().numpy(), cm.cpu().numpy())
        del ws
        t = time.perf_counter()
        want = ce.scipy_lcc(lab, NUM_CLS, conn, gt)
        host_s = time.perf_counter() - t
        same = all(np.array_equal(a, b) for a, b in zip(got, want))
        row = {"volume": name, "shape": list(lab.shape), "connectivity": conn, "kernel_ms": ms, "calls": calls,
               "voxels_per_s": lab.size / ms * 1e3, "scipy_s": host_s, "bit_identical": bool(same),
               "components": want[1][1:, 0].tolist(), "removed": want[1][1:, 2].tolist()}
        print("%-24s %s conn %2d: pnp_largest_components %8.3f ms (%.2f G voxels/s), scipy %7.2f s, components %s, bit-identical %s"
              % (name, "x".join(map(str, lab.shape)), conn, ms, lab.size / ms * 1e-6, host_s, row["components"], same))
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark measures the GPU and needs one"
    import pnp_b200  # noqa: F401
    card, power = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit %s" % (card, power))
    res = {"card": card, "power_limit": power, "classes": NUM_CLS, "runs": []}
    native = native_phantom()
    res["runs"] += measure("native phantom", native, native, a.calls)
    res["runs"] += measure("native phantom + 0.5%", salt(native, 0.005, 1), native, a.calls)
    del native
    base = organs()
    for density, seed in ((0.001, 2), (0.05, 3), (0.31, 4)):
        res["runs"] += measure("organs + %g%%" % (density * 100), salt(base, density, seed), base, a.calls)
    res["all_bit_identical"] = all(r["bit_identical"] for r in res["runs"])
    print("all bit-identical to scipy: %s" % res["all_bit_identical"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
