"""Test-time adaptation of a checkpoint to unlabelled target slices by entropy minimisation (TENT, Wang et al., ICLR 2021).

Every convolution weight stays fixed.  Only the covered batch norms' scales and shifts (gamma, beta) train, with batch-statistics
batch norm in those layers and keep_prob 1, to lower the mean per-pixel softmax entropy of the network's own prediction
(functional.entropy_loss, pnp_entropy_*).  The optimizer is a fresh Adam over the trainer's own arena: the gamma / beta live
there, and every other variable of the arena gets a zero gradient and zero slots, so its update is exactly 0.  After the steps
the covered moving statistics are re-estimated as population statistics of the adapted network (bnstats.py), so the result is
an ordinary inference-mode checkpoint (DESIGN 6.1).

`main` is the command-line tool adapt_entropy.py: checkpoint in, adapted checkpoint and per-step entropy log out."""
import math
import os

import numpy as np
import torch

from . import functional as F
from . import optim
from . import runtime as rt


class EntropyAdaptation:
    """one adaptation session on `trainer`: while it is open only `covered` (the gamma / beta variables) require gradients, and
    a fresh Adam(lr, 0.9, 0.999, 1e-8) without weight decay steps `arena`.  step(x) is one eager step, replay(x) the captured one
    (capture(x) first; eager if the capture failed).  restore() puts back what the session snapshotted on opening -- the covered
    gamma / beta, every batch-norm moving statistic and every requires_grad flag -- bit for bit; close() restores the flags,
    moves the versions of the changed variables and releases the captured steps.  `forward(x)` -> logits; `cache_vars`: the
    variables whose operand caches the step reads; `on_close()` runs at the end of close()."""

    def __init__(self, trainer, arena, covered, forward, lr, cache_vars, on_close=None):
        if trainer.dp.on:
            raise NotImplementedError("entropy adaptation runs on one rank; data-parallel adaptation is not supported")
        lr = float(lr)
        if not (math.isfinite(lr) and lr > 0.0):
            raise ValueError("lr must be positive and finite, got %r" % lr)
        ids = {id(v) for v in arena.vars}
        if not covered or any(id(v) not in ids for v in covered):
            raise ValueError("the covered gamma / beta must all live in the arena")
        self.trainer, self.arena, self.covered, self.forward = trainer, arena, list(covered), forward
        self.cache_vars, self.on_close = list(cache_vars), on_close
        self.batch_size = trainer.net.batch_size
        variables = rt.global_variables()
        self.moving = [v for v in variables if v.pnp_kind == "bn_moving"]
        self._flags = [(v, v.requires_grad) for v in variables]
        self._saved = [(v, v.detach().clone()) for v in self.covered + self.moving]
        for v in variables:
            v.requires_grad_(False)
        for v in self.covered:
            v.requires_grad_(True)
        self.opt = optim.Adam(arena, lr=lr, beta1=0.9, beta2=0.999, eps=1e-8)
        self._one = torch.tensor(1.0, device=arena.theta.device)
        self._graph = None
        self._open = True

    def check_batch(self, x):
        if x.dim() != 4 or x.shape[0] != self.batch_size:
            raise ValueError("adaptation batches must hold the network's batch size %d, got shape %s" % (self.batch_size,
                                                                                                          tuple(x.shape)))

    def _step(self, x):
        self.arena.zero_grad()
        rt.scratch.begin_step()
        loss, pbar = F.entropy_loss(self.forward(x))
        torch.autograd.backward([loss], [self._one])
        self.opt.step()
        return loss.detach(), pbar

    def step(self, x):
        """one eager step on batch x -> (mean entropy, p-bar) on the device, before the update"""
        self.check_batch(x)
        return self._step(x)

    def capture(self, x_example):
        """capture the step as a CUDA graph (nothing runs; the eager steps before it are its warm-up) -> whether it worked"""
        self._graph = rt.capture_step("entropy adaptation", self._step, (x_example,), 1.0, 0, self.cache_vars, (self.arena,),
                                      detach=True)
        return self._graph is not None

    def replay(self, x):
        self.check_batch(x)
        if self._graph is None:
            return self._step(x)
        return self._graph.replay(x)

    def restore(self):
        with torch.no_grad():
            for v, saved in self._saved:
                v.copy_(saved)
                v.pnp_version += 1

    def close(self):
        if not self._open:
            return
        self._open = False
        self._graph = None
        for v, flag in self._flags:
            v.requires_grad_(flag)
        for v in self.covered + self.moving:
            v.pnp_version += 1
        F.drop_operand_caches(self.cache_vars)
        self.trainer.release_graphs()
        if self.on_close is not None:
            self.on_close()


def next_batch(source, dev):
    images, _labels = source.next()             # labels are never a training signal
    return images.to(dev, non_blocking=True) if images.device != dev else images


def adapt(open_session, source, steps, lr, recalibrate_batches, recalibrate):
    """the shared body of both trainers' adapt_entropy: `open_session(lr)` -> an EntropyAdaptation, then `steps` steps on batches
    drawn from `source` (.next() -> (images, labels); labels ignored), the first two eager and the rest replayed from a captured
    step, then `recalibrate(source, recalibrate_batches)` -> (names, slices) of the covered moving statistics.  Anything raising
    -- the source, a non-finite loss (FloatingPointError), the recalibration -- puts every snapshotted variable and flag back
    bit for bit.  -> (covered variable names, history [steps, 1 + C] numpy of (mean entropy, p-bar) per step, slices used)"""
    steps, recalibrate_batches = int(steps), int(recalibrate_batches)
    if steps < 1:
        raise ValueError("steps must be >= 1, got %d" % steps)
    if recalibrate_batches < 1:
        raise ValueError("recalibrate_batches must be >= 1, got %d" % recalibrate_batches)
    session = open_session(lr)
    try:
        dev = rt.device()
        hist = None
        for i in range(steps):
            x = next_batch(source, dev)
            if i < 2:
                loss, pbar = session.step(x)
            else:
                if i == 2:
                    session.check_batch(x)
                    session.capture(x)
                loss, pbar = session.replay(x)
            if hist is None:
                hist = torch.empty(steps, 1 + pbar.numel(), dtype=torch.float32, device=dev)
            hist[i, 0].copy_(loss)
            hist[i, 1:].copy_(pbar)
        history = hist.cpu().numpy()
        if not np.isfinite(history).all():
            bad = int(np.argmax(~np.isfinite(history).all(axis=1)))
            raise FloatingPointError("entropy adaptation: non-finite loss or class probability at step %d" % bad)
        session.close()
        names, rslices = recalibrate(source, recalibrate_batches)
    except BaseException:
        session.restore()
        session.close()
        raise
    names = [v.pnp_name for v in session.covered] + list(names)
    return names, history, steps * session.batch_size + rslices


# ---------------------------------------------------------------------------------------------------------------------------
# command-line tool
# ---------------------------------------------------------------------------------------------------------------------------
def check_args(a, error):
    if not a.out.endswith(".npz"):
        error("--out must name an .npz file")
    if os.path.abspath(a.out) == os.path.abspath(a.checkpoint):
        error("--out must differ from --checkpoint")
    if a.steps < 1:
        error("--steps must be >= 1")
    if not (math.isfinite(a.lr) and a.lr > 0.0):
        error("--lr must be positive")
    if a.batch_size < 1:
        error("--batch-size must be >= 1")
    if a.recalibrate_batches < 1:
        error("--recalibrate-batches must be >= 1")


def build_parser():
    import argparse
    ap = argparse.ArgumentParser(description="adapt a checkpoint to unlabelled slices by test-time entropy minimisation of its "
                                             "batch-norm scales and shifts (TENT), then re-estimate their moving statistics")
    ap.add_argument("--trainer", required=True, choices=["gan", "segmenter"])
    ap.add_argument("--checkpoint", required=True, metavar="IN.npz")
    ap.add_argument("--out", required=True, metavar="OUT.npz")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--volumes", metavar="PAIRS", help="file of `image label` NIfTI pairs: augmented slices drawn on the GPU "
                                                        "(labels only place the crop)")
    src.add_argument("--records", metavar="LIST", help="file listing TFRecord files, one per line (the reference's lists/*_list)")
    ap.add_argument("--steps", type=int, default=100, help="adaptation steps")
    ap.add_argument("--lr", type=float, default=1e-4, help="Adam learning rate")
    ap.add_argument("--batch-size", type=int, default=8, help="slices per step")
    ap.add_argument("--recalibrate-batches", type=int, default=200, help="forward passes re-estimating the moving statistics")
    ap.add_argument("--seed", type=int, default=1234, help="seed of the slice stream")
    return ap


def log_path(out):
    """<OUT stem>_entropy.csv next to OUT.npz"""
    return out[:-len(".npz")] + "_entropy.csv"


def write_log(path, history):
    C = history.shape[1] - 1
    with open(path, "w") as f:
        f.write(",".join(["step", "entropy"] + ["pbar_%d" % c for c in range(C)]) + "\n")
        for i, row in enumerate(history):
            f.write(",".join([str(i)] + ["%.9g" % v for v in row]) + "\n")


def main(argv=None):
    import logging
    from .bnstats import make_source, recalibrated_checkpoint
    from .lib import _save
    from .native import build_trainer
    ap = build_parser()
    a = ap.parse_args(argv)
    check_args(a, ap.error)
    logging.basicConfig(level=logging.INFO)
    trainer = build_trainer(a.trainer, a.checkpoint, a.batch_size)
    source = make_source(a)
    names, history, slices = trainer.adapt_entropy(source, a.steps, lr=a.lr, recalibrate_batches=a.recalibrate_batches)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    _save(recalibrated_checkpoint(trainer), a.out[:-len(".npz")])
    write_log(log_path(a.out), history)
    logging.info("entropy %.6g -> %.6g over %d steps; %d variables adapted over %d slices -> %s"
                 % (history[0, 0], history[-1, 0], len(history), len(names), slices, a.out))
    print(a.out)
    return names, history, slices
