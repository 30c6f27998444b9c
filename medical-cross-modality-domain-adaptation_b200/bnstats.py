"""Re-estimation of batch-norm moving statistics as exact population statistics (PreciseBN; on target-domain slices, AdaBN).

N forward passes run with batch-statistics batch norm on the covered layers and keep_prob 1.  Every covered layer hands the
fp64 per-channel sums its forward computed anyway (functional.layer_forward -> Collector.add); one pnp_bn_accumulate launch
per pass adds them to per-layer fp64 accumulators in pass order, and one pnp_bn_population launch at the end replaces the
moving statistics by the pooled mean and unbiased variance of every value seen (DESIGN 6.1).

`main` is the command-line tool recalibrate_bn.py: checkpoint in, recalibrated checkpoint out."""
import contextlib
import os

import numpy as np
import torch

from . import functional as F
from . import runtime as rt
from ._C import BnAccEntry, BnPopEntry, call, ptr


class Collector:
    """per-layer fp64 accumulators [2C] and host-side counts for the batch norms whose moving statistics are `moving`
    ([(moving_mean, moving_variance)] variables).  Between begin_pass() and end_pass() every covered layer must hand its
    statistics exactly once, with the same M = B * Ho * Wo in every pass."""

    def __init__(self, moving):
        self.moving = list(moving)
        if not self.moving:
            raise ValueError("no batch norm to recalibrate")
        dev = self.moving[0][0].device
        self.index = {mm.pnp_name: i for i, (mm, _) in enumerate(self.moving)}
        self.acc = [torch.zeros(2 * mm.numel(), dtype=torch.float64, device=dev) for mm, _ in self.moving]
        self.M = [None] * len(self.moving)
        self.count = [0] * len(self.moving)
        self.passes = 0
        self._seen = None

    def add(self, bn, stats, M):
        """a covered layer's batch statistics (sum, sumsq) of this pass"""
        name = bn.moving_mean.pnp_name
        i = self.index.get(name)
        if i is None:
            raise RuntimeError("batch-norm recalibration: %s ran with batch statistics but is not covered" % name)
        if self._seen is None:
            raise RuntimeError("batch-norm recalibration: %s ran outside a pass" % name)
        if i in self._seen:
            raise RuntimeError("batch-norm recalibration: %s ran twice in one pass" % name)
        if self.M[i] is not None and self.M[i] != M:
            raise RuntimeError("batch-norm recalibration: %s saw %d values per channel, %d in the earlier passes" % (name, M, self.M[i]))
        self._seen[i] = (stats, M)

    def begin_pass(self):
        self._seen = {}

    def end_pass(self):
        """one pnp_bn_accumulate launch over every covered layer.  The launch reads the pass's statistics buffers on the stream
        after the layers wrote them; a later allocation on the same stream that reuses them is ordered after it."""
        missing = [self.moving[i][0].pnp_name for i in range(len(self.moving)) if i not in self._seen]
        if missing:
            raise RuntimeError("batch-norm recalibration: %d covered batch norms did not run in this pass, e.g. %s" % (len(missing), missing[0]))
        table = (BnAccEntry * len(self.moving))()
        for i, (mm, _) in enumerate(self.moving):
            (s, sq), M = self._seen[i]
            table[i] = BnAccEntry(ptr(s), ptr(sq), ptr(self.acc[i]), mm.numel())
        call("pnp_bn_accumulate", table, len(self.moving), rt.stream())
        for i in range(len(self.moving)):
            M = self._seen[i][1]
            self.M[i] = M
            self.count[i] += M
        self._seen = None
        self.passes += 1

    def finish(self):
        """one pnp_bn_population launch writes every covered statistic; their versions move (folded inference coefficients and
        other operand caches re-derive them)"""
        if self.passes < 1:
            raise RuntimeError("batch-norm recalibration: no pass ran")
        table = (BnPopEntry * len(self.moving))()
        for i, (mm, mv) in enumerate(self.moving):
            table[i] = BnPopEntry(ptr(self.acc[i]), self.count[i], ptr(mm), ptr(mv), mm.numel())
        call("pnp_bn_population", table, len(self.moving), rt.stream())
        for mm, mv in self.moving:
            mm.pnp_version += 1
            mv.pnp_version += 1


def covered_statistics(variables):
    """[(moving_mean, moving_variance)] of the batch-norm scopes among `variables`, in graph order"""
    by_name = {v.pnp_name: v for v in variables}
    out = []
    for v in variables:
        if v.pnp_name.endswith("/moving_mean"):
            out.append((v, by_name[v.pnp_name[:-len("moving_mean")] + "moving_variance"]))
    return out


@contextlib.contextmanager
def collecting(moving):
    """a Collector over `moving`, active in functional.layer_forward inside the block.  The covered statistics are snapshotted on
    entry and put back bit for bit if the block raises (its training-mode passes move them through the 0.9 update)."""
    if F.BN_COLLECTOR is not None:
        raise RuntimeError("batch-norm recalibration: a collection is already active")
    col = Collector(moving)
    saved = [(mm.detach().clone(), mv.detach().clone()) for mm, mv in col.moving]
    F.BN_COLLECTOR = col
    try:
        yield col
    except BaseException:
        with torch.no_grad():
            for (mm, mv), (a, b) in zip(col.moving, saved):
                mm.copy_(a)
                mv.copy_(b)
                mm.pnp_version += 1
                mv.pnp_version += 1
        raise
    finally:
        F.BN_COLLECTOR = None


def recalibrate(trainer, source, batches, moving, forward):
    """the shared body of both trainers' recalibrate_bn: `batches` passes of `forward(x)` on images drawn from `source`
    (.next() -> (images, labels); labels ignored) -> (covered variable names, slice count)"""
    if trainer.dp.on:
        raise NotImplementedError("batch-norm recalibration runs on one rank; data-parallel recalibration is not supported")
    batches = int(batches)
    if batches < 1:
        raise ValueError("batches must be >= 1, got %d" % batches)
    B = trainer.net.batch_size
    dev = rt.device()
    slices = 0
    with collecting(moving) as col, torch.no_grad():
        for _ in range(batches):
            images, _labels = source.next()
            x = images.to(dev, non_blocking=True) if images.device != dev else images
            if x.dim() != 4 or x.shape[0] != B:
                raise ValueError("recalibration batches must hold the network's batch size %d, got shape %s" % (B, tuple(x.shape)))
            rt.scratch.begin_step()
            col.begin_pass()
            forward(x)
            col.end_pass()
            slices += B
        col.finish()
    trainer.release_graphs()          # captured steps hold folded coefficients of the old statistics
    names = []
    for mm, mv in moving:
        names += [mm.pnp_name, mv.pnp_name]
    return names, slices


# ---------------------------------------------------------------------------------------------------------------------------
# command-line tool
# ---------------------------------------------------------------------------------------------------------------------------
def recalibrated_checkpoint(trainer):
    """every graph variable (the recalibrated statistics as they now are) and pnp/global_step of the input checkpoint; no
    optimizer slot and no EMA key"""
    st = rt.state_dict()
    d = getattr(trainer.net, "last_restored", None) or {}
    st["pnp/global_step"] = np.int64(d.get("pnp/global_step", 0))
    return st


def check_args(a, error):
    if not a.out.endswith(".npz"):
        error("--out must name an .npz file")
    if os.path.abspath(a.out) == os.path.abspath(a.checkpoint):
        error("--out must differ from --checkpoint")
    if a.scope is not None and a.trainer != "gan":
        error("--scope applies to --trainer gan")
    if a.batches < 1:
        error("--batches must be >= 1")
    if a.batch_size < 1:
        error("--batch-size must be >= 1")


def build_parser():
    import argparse
    ap = argparse.ArgumentParser(description="re-estimate a checkpoint's batch-norm moving statistics as exact population "
                                             "statistics over many slices (PreciseBN; AdaBN on target-domain slices)")
    ap.add_argument("--trainer", required=True, choices=["gan", "segmenter"])
    ap.add_argument("--checkpoint", required=True, metavar="IN.npz")
    ap.add_argument("--out", required=True, metavar="OUT.npz")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--volumes", metavar="PAIRS", help="file of `image label` NIfTI pairs: augmented slices drawn on the GPU")
    src.add_argument("--records", metavar="LIST", help="file listing TFRecord files, one per line (the reference's lists/*_list)")
    ap.add_argument("--batches", type=int, default=200, help="forward passes")
    ap.add_argument("--batch-size", type=int, default=8, help="slices per pass")
    ap.add_argument("--scope", choices=["dam", "all"], default=None,
                    help="gan: the DAM's batch norms (default), or also the shared groups 7-9")
    ap.add_argument("--seed", type=int, default=1234, help="seed of the slice stream")
    return ap


def make_source(a):
    if a.volumes:
        from .train_segmenter import volume_source
        return volume_source(a.volumes, a.batch_size, a.seed)
    from .lib import _read_lists
    from .tfrecord import TFRecordSource
    files = _read_lists(a.records)
    if not files:
        raise SystemExit("no TFRecord files listed in %s" % a.records)
    return TFRecordSource(files, a.batch_size, seed=a.seed)


def main(argv=None):
    import logging
    from .lib import _save
    from .native import build_trainer
    ap = build_parser()
    a = ap.parse_args(argv)
    check_args(a, ap.error)
    logging.basicConfig(level=logging.INFO)
    trainer = build_trainer(a.trainer, a.checkpoint, a.batch_size)
    source = make_source(a)
    if a.trainer == "gan":
        names, slices = trainer.recalibrate_bn(source, a.batches, scope=a.scope or "dam")
    else:
        names, slices = trainer.recalibrate_bn(source, a.batches)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    _save(recalibrated_checkpoint(trainer), a.out[:-len(".npz")])
    logging.info("recalibrated %d batch-norm statistics over %d slices -> %s" % (len(names), slices, a.out))
    print(a.out)
    return names, slices
