"""Throughput of the TFRecord input pipeline (SURVEY 8f #2) on the host cores: examples/s and GB/s of decoded fp32 images
for 1 / 4 / 8 / 16 reader threads, CRC check on, files in the page cache (tmpfs when available).  The 8-GPU adversarial step at
~800 slices/s/GPU consumes 3 slices of 786 KB per step per GPU-slot: ~5 GB/s for the whole box.

    python scripts/bench_input_pipeline.py [--files 64] [--seconds 3] [--out result.json]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import pnp_b200  # noqa: F401
    from pnp_b200 import tfrecord as tfr, _io
    base = "/dev/shm" if os.path.isdir("/dev/shm") and os.access("/dev/shm", os.W_OK) else None
    d = tempfile.mkdtemp(prefix="pnp_tfr_", dir=base)
    try:
        rng = np.random.RandomState(0)
        files = []
        for i in range(a.files):
            img = rng.randn(256, 256, 3).astype(np.float32)
            lab = rng.randint(0, 5, (256, 256, 3)).astype(np.float32)
            p = os.path.join(d, "s%04d.tfrecords" % i)
            tfr.write_record(p, [tfr.encode_example(img, lab)])
            files.append(p)
        file_bytes = os.path.getsize(files[0])
        res = {"crc32c_hardware": bool(_io.lib.pnp_crc32c_is_hardware()), "host_cores": os.cpu_count(), "file_bytes": file_bytes,
               "image_bytes_per_example": 256 * 256 * 3 * 4, "batch": a.batch, "where": d, "runs": []}
        # raw CRC speed of one core
        buf = open(files[0], "rb").read()
        t0 = time.time()
        n = 0
        while time.time() - t0 < 0.5:
            _io.lib.pnp_crc32c(buf, len(buf))
            n += 1
        res["crc32c_gbs_one_core"] = n * len(buf) / (time.time() - t0) / 1e9
        for threads in (0, 1, 4, 8, 16):
            src = tfr.TFRecordSource(files, a.batch, seed=1, num_threads=threads)
            src.next()
            t0 = time.time()
            nb = 0
            while time.time() - t0 < a.seconds:
                src.next()
                nb += 1
            dt = time.time() - t0
            src.close()
            ex = nb * a.batch / dt
            run = {"reader_threads": threads, "examples_per_s": ex, "decoded_image_GBps": ex * 256 * 256 * 3 * 4 / 1e9,
                   "file_GBps": ex * file_bytes / 1e9}
            print(run, flush=True)
            res["runs"].append(run)
        if a.out:
            with open(a.out, "w") as f:
                json.dump(res, f, indent=1)
        print(json.dumps({k: v for k, v in res.items() if k != "runs"}))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
