"""Exponential moving average of the trained weights: tf.train.ExponentialMovingAverage(decay, num_updates=n) over an optimizer
arena and a list of further variables (the batch-norm moving statistics), kept in one flat shadow buffer and advanced by two
launches per optimizer step (elementwise.cu: pnp_ema_advance, pnp_ema_update).

The average never feeds back into training: it reads the live variables and writes only its own buffer, count and factor.
Checkpoints store each shadow under TF's name '<variable>/ExponentialMovingAverage', and `averaged_weights` turns such a
checkpoint into an ordinary one whose variables are the averages (lib.save_checkpoint writes it next to every checkpoint)."""
import contextlib

import numpy as np
import torch

from . import runtime as rt
from ._C import call, ptr
from .optim import CHUNK

SUFFIX = "/ExponentialMovingAverage"
NUM_UPDATES_KEY = "pnp/ema_num_updates"
DECAY_KEY = "pnp/ema_decay"


def check_decay(decay):
    decay = float(decay)
    if not 0.0 < decay < 1.0:
        raise ValueError("EMA decay must lie in (0, 1), got %r" % decay)
    return decay


class EMA:
    """Shadow of `arena` (optim.Arena, mirrored float for float) and of `extra` (contiguous fp32 variables outside the arena,
    one 1024-float-padded segment each, reached through a device table of (live pointer, length) per chunk).  The table
    holds the extra variables' storage addresses: they must be updated in place (copy_, all_reduce), never rebound."""

    def __init__(self, arena, extra, decay):
        self.decay = check_decay(decay)
        self.arena = arena
        self.extra = list(extra)
        dev = arena.theta.device
        entries, self.extra_offsets, off = [], [], arena.total
        for v in self.extra:
            if v.dtype != torch.float32 or not v.is_contiguous() or v.device != dev:
                raise ValueError("EMA: %s is not a contiguous fp32 tensor on %s" % (getattr(v, "pnp_name", "?"), dev))
            n = v.numel()
            self.extra_offsets.append(off)
            for j in range(0, n, CHUNK):
                entries.append((v.data_ptr() + 4 * j, min(CHUNK, n - j)))
                off += CHUNK
        self.total = off
        self.table_n = len(entries)
        self.table = torch.tensor(entries, dtype=torch.int64, device=dev).reshape(-1, 2) if entries else None   # pnp_ema_chunk[]
        self.shadow = torch.zeros(off, dtype=torch.float32, device=dev)
        self.num_updates = torch.zeros(1, dtype=torch.int64, device=dev)
        self.c = torch.zeros(1, dtype=torch.float32, device=dev)
        self.init_from_live()

    def _pairs(self):
        """(variable, its shadow view) for every covered variable, arena first"""
        out = [(v, self.shadow[o:o + n].view(v.shape)) for v, (o, n) in zip(self.arena.vars, self.arena.offsets)]
        out += [(v, self.shadow[o:o + v.numel()].view(v.shape)) for v, o in zip(self.extra, self.extra_offsets)]
        return out

    @property
    def variables(self):
        return self.arena.vars + self.extra

    def init_from_live(self):
        """every shadow := its live variable, n := 0"""
        with torch.no_grad():
            self.shadow[:self.arena.total].copy_(self.arena.theta)
            for v, s in self._pairs()[len(self.arena.vars):]:
                s.copy_(v)
            self.num_updates.zero_()

    def update(self):
        """one averaged step (captured graphs record both launches)"""
        call("pnp_ema_advance", ptr(self.num_updates), self.decay, ptr(self.c), rt.stream())
        call("pnp_ema_update", ptr(self.shadow), ptr(self.arena.theta), self.arena.total, ptr(self.table), self.table_n, ptr(self.c),
             rt.stream())

    def _swap(self):
        call("pnp_ema_swap", ptr(self.shadow), ptr(self.arena.theta), self.arena.total, ptr(self.table), self.table_n, rt.stream())
        for v in self.variables:            # cached operand planes and folded batch-norm coefficients key on the versions
            v.pnp_version += 1

    @contextlib.contextmanager
    def swapped(self):
        """the shadows are the live variables inside the block (contents exchanged bit for bit, and back on leaving)"""
        self._swap()
        try:
            yield self
        finally:
            self._swap()

    def average_over_ranks(self, dp):
        """the batch-norm shadows' mean over the data-parallel ranks, in place (DataParallel.average_moving_stats does the same
        for the live statistics).  The arena shadows are equal on every rank already, as the live arena is."""
        if not dp.on or self.total == self.arena.total:
            return
        import torch.distributed as dist
        stats = self.shadow[self.arena.total:]
        dist.all_reduce(stats, op=dist.ReduceOp.SUM)
        stats.mul_(1.0 / dp.world)

    def state(self):
        """checkpoint keys: '<var>/ExponentialMovingAverage' per covered variable, the update count and the decay"""
        d = {v.pnp_name + SUFFIX: s.detach().cpu().numpy().copy() for v, s in self._pairs()}
        d[NUM_UPDATES_KEY] = np.int64(self.num_updates.item())
        d[DECAY_KEY] = np.float32(self.decay)
        return d

    def load_state(self, d):
        """load the shadows and the count of a checkpoint that holds them -> whether it did (the decay in use is kept)"""
        if NUM_UPDATES_KEY not in d:
            return False
        pairs = self._pairs()
        missing = [v.pnp_name for v, _ in pairs if v.pnp_name + SUFFIX not in d]
        if missing:
            raise KeyError("checkpoint holds EMA state but no shadow of %s" % missing[:5])
        with torch.no_grad():
            for v, s in pairs:
                s.copy_(torch.as_tensor(np.asarray(d[v.pnp_name + SUFFIX]), dtype=s.dtype).reshape(s.shape))
            self.num_updates.fill_(int(d[NUM_UPDATES_KEY]))
        return True


def averaged_weights(state, names):
    """the averaged-weights checkpoint of a checkpoint `state` with EMA keys: every variable of `names`, its shadow where it has
    one, and pnp/global_step; no optimizer slot and no EMA key"""
    out = {n: state.get(n + SUFFIX, state[n]) for n in names}
    out["pnp/global_step"] = state["pnp/global_step"]
    return out
