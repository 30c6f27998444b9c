"""Data parallelism for the hot path: one process per GPU, parameters and optimizer state replicated,
the per-slice minibatch sharded across ranks, and ONE all-reduce (NCCL over NVLink/NVSwitch, or gloo in
the CPU tests) over the flat gradient arena per optimizer step.  The 1/N average is folded into the
optimizer kernel (`grad_scale`), so no extra pass touches the gradients.

The reference is single-GPU (train_segmenter.py:20, train_gan.py:18); parity under DP is defined as:
an N-rank step == the average of N single-GPU reference steps at the per-rank batch (batch-norm
statistics, the CE class weights and the Dice sums stay per rank -- SURVEY 8e).
"""
import os
import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """Initialise torch.distributed from the torchrun environment (RANK / WORLD_SIZE / MASTER_*)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1 or dist.is_initialized():
        return
    if backend is None:
        backend = "nccl" if torch.cuda.is_available() else "gloo"
    if backend == "nccl":     # a gloo group (CPU tensors) must not claim a GPU per rank: ranks may outnumber the GPUs
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    import datetime
    # a rank that stops participating must abort the job quickly instead of hanging the box
    dist.init_process_group(backend=backend, timeout=datetime.timedelta(seconds=int(os.environ.get("PNP_DIST_TIMEOUT", "180"))))


class BucketedAllReduce:
    """The gradient all-reduce of one arena, started bucket by bucket DURING the backward pass (SURVEY 8e: "bucketed in
    reverse-layer order to overlap with the remaining backward").  The arena is laid out in variable-creation (= forward) order,
    so the backward pass completes it from the back: it is cut into `n_buckets` contiguous ranges on variable boundaries, every
    gradient contribution (weight-gradient launch, BN dgamma/dbeta, FC) reports through `contribution(var)`, and a bucket whose
    variables have all received the number of contributions the first (calibration) step saw is handed to NCCL with
    async_op=True: the collective waits for the compute stream's position at that moment and then runs beside the rest of
    the backward.  `finish()` makes the compute stream wait for all of them.  Step structure is fixed per arena (D step / G
    step / segmenter step), so the calibration holds; a step that deviates raises instead of reducing a half-written bucket."""

    def __init__(self, arena, n_buckets=4):
        self.arena = arena
        self.grad = arena.grad
        n = len(arena.vars)
        target = arena.total / float(max(1, n_buckets))
        self.bounds, self.bucket_of = [], {}
        lo_var, lo_off, acc = 0, 0, 0
        for i, (v, (o, cnt)) in enumerate(zip(arena.vars, arena.offsets)):
            end = arena.offsets[i + 1][0] if i + 1 < n else arena.total
            acc = end - lo_off
            if acc >= target or i == n - 1:
                self.bounds.append((lo_off, end))
                for j in range(lo_var, i + 1):
                    self.bucket_of[id(arena.vars[j])] = len(self.bounds) - 1
                lo_var, lo_off = i + 1, end
        self.expected = None              # per variable: contributions per step, learned in the first (calibration) step
        self.calibrating = False
        self.passive = False
        self.handles = []
        self.begin()

    def begin(self, passive=False):
        """passive: count only -- the caller wants the LOCAL gradients first (d_step(apply=False)); finish() then reduces in one call"""
        self.var_count = {}
        self.launched = [False] * len(self.bounds)
        self.handles = []
        self.calibrating = self.expected is None
        self.passive = bool(passive)
        if not self.calibrating:
            # variables that still owe contributions, per bucket
            self.pending = [0] * len(self.bounds)
            for vid, n in self.expected.items():
                if n > 0:
                    self.pending[self.bucket_of[vid]] += 1

    def contribution(self, var):
        vid = id(var)
        b = self.bucket_of.get(vid)
        if b is None:
            return
        c = self.var_count.get(vid, 0) + 1
        self.var_count[vid] = c
        if self.calibrating:
            return
        want = self.expected.get(vid, 0)
        if c > want:
            raise RuntimeError("bucketed all-reduce: %s received more gradient contributions than the calibration step (%d > %d)"
                               % (getattr(var, "pnp_name", "variable"), c, want))
        if c == want:
            self.pending[b] -= 1
            if self.pending[b] == 0 and not self.passive and not self.launched[b]:
                lo, hi = self.bounds[b]
                self.handles.append(dist.all_reduce(self.grad[lo:hi], op=dist.ReduceOp.SUM, async_op=True))
                self.launched[b] = True

    def finish(self):
        if self.calibrating:
            self.expected = dict(self.var_count)
        if self.calibrating or self.passive:
            dist.all_reduce(self.grad, op=dist.ReduceOp.SUM)
            return
        for b, (lo, hi) in enumerate(self.bounds):
            if not self.launched[b]:
                if self.pending[b] != 0 and any(self.var_count.get(vid, 0) for vid, bb in self.bucket_of.items() if bb == b):
                    raise RuntimeError("bucketed all-reduce: bucket %d is missing gradient contributions of %d variables" % (b, self.pending[b]))
                self.handles.append(dist.all_reduce(self.grad[lo:hi], op=dist.ReduceOp.SUM, async_op=True))
        for h in self.handles:
            h.wait()
        self.handles = []


class DataParallel:
    def __init__(self):
        self.on = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        self.world = dist.get_world_size() if self.on else 1
        self.rank = dist.get_rank() if self.on else 0

    def allreduce(self, grad_arena):
        """sum-all-reduce the flat gradient arena in place; returns the grad_scale (1/world) to hand to
        the optimizer kernel."""
        if self.on:
            dist.all_reduce(grad_arena, op=dist.ReduceOp.SUM)
        return 1.0 / self.world

    # ---- overlapped variant -----------------------------------------------------------------------------------------------
    def attach(self, arena, n_buckets=None):
        """bucketed, overlapped all-reduce for this arena (no-op on one rank; PNP_DP_BUCKETS=0 keeps the single call)"""
        if n_buckets is None:
            n_buckets = int(os.environ.get("PNP_DP_BUCKETS", "4"))
        if not self.on or n_buckets <= 0:
            return None
        red = BucketedAllReduce(arena, n_buckets)
        for v in arena.vars:
            v._pnp_grad_hook = red.contribution
        arena._pnp_reducer = red
        return red

    def begin_backward(self, arena, overlap=True):
        red = getattr(arena, "_pnp_reducer", None)
        if red is not None:
            red.begin(passive=not overlap)

    def finish_backward(self, arena):
        """-> grad_scale.  With an attached reducer: wait for the bucket collectives started during the backward pass."""
        red = getattr(arena, "_pnp_reducer", None)
        if red is None:
            return self.allreduce(arena.grad)
        red.finish()
        return 1.0 / self.world

    def broadcast_params(self, theta_arena):
        """make every replica start from rank 0's parameters"""
        if self.on:
            dist.broadcast(theta_arena, src=0)

    def barrier(self):
        if self.on:
            dist.barrier()

    def broadcast_variables(self, variables):
        """every replica continues from rank 0's values: ALL graph variables (frozen weights and BN moving statistics
        included), after construction and after every restore -- replicas must not depend on identical host seeds"""
        if not self.on:
            return
        seen = set()
        with torch.no_grad():
            for v in variables:
                arena = getattr(v, "_pnp_arena", None)
                t = arena.theta if arena is not None else v
                if id(t) in seen:
                    continue
                seen.add(id(t))
                dist.broadcast(t, src=0)
                if arena is None:
                    v.pnp_version = getattr(v, "pnp_version", 0) + 1
        for v in variables:
            if getattr(v, "_pnp_arena", None) is not None:
                v.pnp_version = getattr(v, "pnp_version", 0) + 1

    def average_moving_stats(self, variables):
        """BN moving statistics are updated from per-rank batches (SURVEY 8e: no SyncBN); a checkpoint stores their mean"""
        if not self.on:
            return
        with torch.no_grad():
            for v in variables:
                if getattr(v, "pnp_kind", "") == "bn_moving":
                    dist.all_reduce(v, op=dist.ReduceOp.SUM)
                    v.mul_(1.0 / self.world)
                    v.pnp_version = getattr(v, "pnp_version", 0) + 1

    def save_checkpoint(self, save_fn):
        """rank 0 alone writes (save_fn must write atomically); every rank waits for the file to be complete"""
        if self.rank == 0:
            save_fn()
        self.barrier()
