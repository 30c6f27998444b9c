"""The coherence audit of the host-side operand state: every cached operand of a registered variable (bf16 weight planes,
transposed SIMT weights, folded inference-mode batch-norm coefficients) that claims to be current is re-derived from the live
values with the same C-ABI call and compared bit for bit, and every activation whose bf16 planes travel as an attribute is
re-split at the moment a consumer trusts them.  The three kernels behind the caches are pinned by test_tc_split_exact_gpu.py,
test_simt_exact_gpu.py and test_elementwise_exact_gpu.py, so "equal to a fresh call" is "equal to the reference".

A helper module: no tests in it.  It imports without a GPU."""
import contextlib
import sys

import torch

from tests import cabi

BN_LEAVES = ("gamma", "beta", "moving_mean", "moving_variance")      # the order of functional._bn_infer_coef's key


def _same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def bn_scope_vars(rt, gamma_name):
    """the four variables of the batch norm whose gamma is `gamma_name`, in the order of the coefficient cache's key"""
    scope = gamma_name[:-len("/gamma")]
    return [rt.graph.vars["%s/%s" % (scope, leaf)] for leaf in BN_LEAVES]


def bn_key(rt, gamma_name):
    return tuple(v.pnp_version for v in bn_scope_vars(rt, gamma_name))


def audit(rt, F):
    """-> {"planes", "wT", "bncoef": live entries re-derived and found equal, "stale": entries with an older stamp, skipped};
    raises AssertionError naming the variable of the first live entry that is not what a fresh call makes of the live values"""
    from pnp_b200 import _C
    n = {"planes": 0, "wT": 0, "bncoef": 0, "stale": 0}
    for name, v in rt.graph.vars.items():
        ver = v.pnp_version
        planes = v.__dict__.get("_pnp_planes")
        for key, (stamp, hi, lo) in (planes.items() if isinstance(planes, dict) else ()):
            if stamp != ver:
                n["stale"] += 1
                continue
            for_dgrad, nterms, cin_pad = key
            rh, rl = cabi.split_w_dev(_C, rt, v.detach(), for_dgrad, nterms, cin_pad)
            assert _same_bits(hi, rh) and _same_bits(lo, rl), \
                "%s: cached bf16 weight planes %r carry the current version %d but are not the split of the live weights" % (name, key, ver)
            n["planes"] += 1
        hit = v.__dict__.get("_pnp_wT")
        if hit is not None:
            if hit[0] != ver:
                n["stale"] += 1
            else:
                kh, kw, cin, cout = v.shape
                ref = torch.empty(kh, kw, cout, cin, dtype=v.dtype, device=v.device)
                _C.call("pnp_weight_transpose", _C.ptr(v), _C.ptr(ref), kh * kw, cin, cout, rt.stream())
                assert _same_bits(hit[1], ref), \
                    "%s: cached transposed weights carry the current version %d but are not the transpose of the live weights" % (name, ver)
                n["wT"] += 1
        hit = v.__dict__.get("_pnp_bncoef")
        if hit is not None:
            assert name.endswith("/gamma"), "%s: batch-norm coefficients cached on a variable that is not a gamma" % name
            key, vec = hit
            assert len(key) == 4, (name, key)
            if tuple(key) != bn_key(rt, name):
                n["stale"] += 1
            else:
                g, b, mm, mv = bn_scope_vars(rt, name)
                C = g.numel()
                ref = torch.empty(4, C, dtype=torch.float32, device=g.device)
                _C.call("pnp_bn_finalize", None, None, 1, C, _C.ptr(g), _C.ptr(b), _C.ptr(mm), _C.ptr(mv), 0, _C.ptr(ref[0]),
                        _C.ptr(ref[1]), _C.ptr(ref[2]), _C.ptr(ref[3]), rt.stream())
                assert _same_bits(vec, ref), \
                    "%s: folded batch-norm coefficients are keyed %r, the current versions, but are not those of the live " \
                    "gamma / beta / moving statistics" % (name, tuple(key))
                n["bncoef"] += 1
    return n


def cache_fingerprint(rt):
    """{(variable, kind, key): (stamp, address)} of every cache entry: equal fingerprints mean nothing was re-derived"""
    out = {}
    for name, v in rt.graph.vars.items():
        planes = v.__dict__.get("_pnp_planes")
        for key, (stamp, hi, lo) in (planes.items() if isinstance(planes, dict) else ()):
            out[(name, "planes", key)] = (stamp, hi.data_ptr())
        hit = v.__dict__.get("_pnp_wT")
        if hit is not None:
            out[(name, "wT", None)] = (hit[0], hit[1].data_ptr())
        hit = v.__dict__.get("_pnp_bncoef")
        if hit is not None:
            out[(name, "bncoef", None)] = (tuple(hit[0]), hit[1].data_ptr())
    return out


def drop_caches(rt):
    """forget every cached operand, so that the next use re-derives it from the live values: the cold-cache control"""
    for v in rt.graph.vars.values():
        for attr in ("_pnp_planes", "_pnp_wT", "_pnp_bncoef"):
            v.__dict__.pop(attr, None)


class PlaneWatch:
    def __init__(self):
        self.hits, self.mismatches = 0, []


@contextlib.contextmanager
def watch_planes(F):
    """Inside the block every activation whose attached bf16 planes a consumer is about to trust is split again from its
    current fp32 values; on exit an AssertionError lists the call sites (function and layer tag) where the two differ.
    `_PlanesOnly` objects have no fp32 values and are skipped.  Every check synchronises: eager code only, never in a capture.
    Only `functional._planes_of` is watched: the planes of a layer's input that the forward pass saves for its weight gradient
    (`saved["xs"]`) are handed over without it, so a write to that input between forward and backward is not seen here."""
    w = PlaneWatch()
    inner = F._planes_of

    def checked(x, nterms):
        p = getattr(x, "_pnp_planes", None)
        if p is not None and p[0] == nterms and isinstance(x, torch.Tensor):
            w.hits += 1
            hi, lo = F.split_bf16(x.detach(), nterms)
            if not (_same_bits(p[1], hi) and _same_bits(p[2], lo)):
                fr = sys._getframe(1)
                g = fr.f_locals.get("geom")
                tag = "?" if g is None else "%dx%d.%d.%d.k%ds%d" % (g.Ho, g.Wo, g.Cin, g.Cout, g.kh, g.stride)
                w.mismatches.append("%s %s" % (fr.f_code.co_name, tag))
        return inner(x, nterms)

    F._planes_of = checked
    try:
        yield w
    finally:
        F._planes_of = inner
    assert not w.mismatches, "attached bf16 planes are not the split of the tensor's current values at: %s" % ", ".join(w.mismatches)
