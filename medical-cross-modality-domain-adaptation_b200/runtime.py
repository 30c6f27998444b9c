"""Process-wide runtime state of the H100 hot path: device, stream, dropout RNG, conv backend choice,
and the TF-style variable registry (names follow the reference's checkpoint naming contract,
lists/half_zip_*_vars, lists/*_bn_list)."""
import contextlib
import os
import torch

from . import _C


# ------------------------------------------------------------------------------------------------
# device / stream
# ------------------------------------------------------------------------------------------------
def device():
    if torch.cuda.is_available():
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")  # host-logic tests only; kernels cannot run here


def stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------
# conv backend: "auto" = wgmma (3-term bf16 split) where eligible, SIMT fp32 elsewhere
#               "simt" = SIMT fp32 everywhere;  "tc1" = wgmma single bf16 term (BASELINE config 5)
# ------------------------------------------------------------------------------------------------
_conv_backend = os.environ.get("PNP_CONV_BACKEND", "auto")


def set_conv_backend(name):
    global _conv_backend
    assert name in ("auto", "simt", "tc3", "tc1")
    _conv_backend = name


def conv_backend():
    return _conv_backend


_tc_ok = None


def tc_available():
    global _tc_ok
    if _tc_ok is None:
        _tc_ok = bool(torch.cuda.is_available() and _C.lib.pnp_tc_available())
    return _tc_ok


# ------------------------------------------------------------------------------------------------
# dropout RNG: the seed lives in device memory (graph-capturable); every dropout call site draws a
# fresh stream id
# ------------------------------------------------------------------------------------------------
class _Rng:
    def __init__(self):
        self.seed_t = None
        self.counter = 0

    def seed(self, s):
        self.seed_t = torch.tensor([int(s) & 0x7FFFFFFFFFFFFFFF], dtype=torch.int64, device=device())
        self.counter = 0

    def seed_ptr(self):
        if self.seed_t is None:
            self.seed(0x5EED)
        return self.seed_t.data_ptr()

    def next_stream(self):
        self.counter += 1
        return self.counter

    def advance(self):
        _C.call("pnp_seed_advance", self.seed_ptr(), stream())


rng = _Rng()


def manual_seed(s):
    rng.seed(s)


# ------------------------------------------------------------------------------------------------
# per-step scratch: zeroed fp64 accumulators (batch-norm sums, loss partials).  A layer takes a slice; the trainers call
# begin_step() once per optimizer step, which re-zeroes exactly what the previous step used with ONE fill kernel (r1: 187 fill
# launches per step).  Slices are 128-byte aligned so that two layers' atomics never share a cache line.
# ------------------------------------------------------------------------------------------------
class Scratch:
    CAP = 1 << 20            # doubles (8 MB)

    def __init__(self):
        self.buf, self.off, self.high = None, 0, 0

    def take(self, n, dev):
        if self.buf is None or self.buf.device != dev:
            if not torch.cuda.is_available():
                return None
            self.buf = torch.zeros(self.CAP, dtype=torch.float64, device=dev)
            self.off = self.high = 0
        n16 = -(-n // 16) * 16
        if self.off + n16 > self.CAP:
            return None
        t = self.buf[self.off:self.off + n]
        self.off += n16
        self.high = max(self.high, self.off)
        return t

    def begin_step(self):
        """everything handed out so far belongs to finished work (same stream): zero it again and start over"""
        if self.buf is not None and self.high > 0:
            _C.call("pnp_fill", self.buf.data_ptr(), 0.0, 2 * self.high, stream())
        self.off = self.high = 0


scratch = Scratch()


# ------------------------------------------------------------------------------------------------
# TF-1.x style variable registry and scopes
# ------------------------------------------------------------------------------------------------
class _Graph:
    def __init__(self):
        self.reset()

    def reset(self):
        self.vars = {}            # name -> tensor
        self.order = []           # creation order
        self.var_scope = []       # tf.variable_scope stack
        self.name_scope = []      # tf.name_scope stack (variable_scope pushes here too)
        self.uniq = {}            # (name-scope prefix, base) -> count, for tf.Variable / default BN scopes
        self.collections = {}


graph = _Graph()


def reset_default_graph():
    graph.reset()


@contextlib.contextmanager
def variable_scope(name, reuse=None):
    """tf.variable_scope: also opens a name scope of the same name ('' opens neither)."""
    if name:
        graph.var_scope.append(name)
        graph.name_scope.append(name)
    try:
        yield name
    finally:
        if name:
            graph.var_scope.pop()
            graph.name_scope.pop()


@contextlib.contextmanager
def root_scope():
    """Temporarily leave every open variable/name scope (names created inside are absolute)."""
    vs, ns = graph.var_scope, graph.name_scope
    graph.var_scope, graph.name_scope = [], []
    try:
        yield
    finally:
        graph.var_scope, graph.name_scope = vs, ns


@contextlib.contextmanager
def name_scope(name):
    graph.name_scope.append(name)
    try:
        yield name
    finally:
        graph.name_scope.pop()


def _unique(prefix, base):
    key = (prefix, base)
    n = graph.uniq.get(key, 0)
    graph.uniq[key] = n + 1
    return base if n == 0 else "%s_%d" % (base, n)


def _register(name, t, trainable, kind):
    t.pnp_name = name
    t.pnp_trainable = bool(trainable)
    t.pnp_kind = kind          # 'weight' | 'bn_gamma' | 'bn_beta' | 'bn_moving'
    t.pnp_version = 0          # bumped whenever the values change (optimizer step / load)
    graph.vars[name] = t
    graph.order.append(name)
    return t


def new_variable(init, trainable=True, kind="weight"):
    """tf.Variable(initial): name 'Variable' uniquified inside the current *name* scope."""
    prefix = "/".join(graph.name_scope)
    leaf = _unique(prefix, "Variable")
    name = (prefix + "/" if prefix else "") + leaf
    return _register(name, init, trainable, kind)


def get_variable(name, make, trainable=True, kind="weight"):
    """tf.get_variable(name) with AUTO_REUSE semantics inside the current *variable* scope."""
    prefix = "/".join(graph.var_scope)
    full = (prefix + "/" if prefix else "") + name
    if full in graph.vars:
        return graph.vars[full]
    return _register(full, make(), trainable, kind)


def default_scope_name(base):
    """tf.variable_scope(None, default_name=base): uniquified inside the current variable scope."""
    prefix = "/".join(graph.var_scope)
    return _unique("vs:" + prefix, base)


def global_variables():
    return [graph.vars[n] for n in graph.order]


def state_dict():
    return {n: graph.vars[n].detach().cpu().numpy().copy() for n in graph.order}


def load_state_dict(d, strict=True):
    """Load numpy arrays keyed by TF variable names (with or without the ':0' suffix)."""
    import numpy as np
    missing = []
    with torch.no_grad():
        for k, v in d.items():
            k = k[:-2] if k.endswith(":0") else k
            if k not in graph.vars:
                missing.append(k)
                continue
            t = graph.vars[k]
            t.copy_(torch.as_tensor(np.asarray(v), dtype=t.dtype).reshape(t.shape))
            t.pnp_version += 1
    if strict and missing:
        raise KeyError("unknown variables: %s" % missing[:5])
    return missing
