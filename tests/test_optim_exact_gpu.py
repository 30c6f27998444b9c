"""The optimizer steps of elementwise.cu (pnp_adam_advance, pnp_adam_step, pnp_rmsprop_step, pnp_momentum_step) against the fp64
references of oracle/optim_exact.py, called at the C-ABI.

a. exact cases: dyadic operands on which every intermediate of the step is an fp32 value (the reference asserts it first), so
   every output equals the reference bit for bit (torch.equal): segment tables with ~300 non-monotone, repeated ids, segments
   with g = 0, grad_scale 1 / 0.5 / 0.25, n = 1024, 3 * 1024 and 2^24, RMSProp theta on and beyond +-clip, clip = 0 segments
   and seg_clip = NULL; the state of pnp_adam_advance over 50 steps bit for bit;
b. real-valued cases at the TF defaults, after several steps: |got - ref| <= TAU * magnitude per element (and the first-order
   gamma bound), with segments whose second moment is of the order of eps;
c. optim.Arena with variable sizes 1, 1023, 1024, 1025 and 3 * 3 * 512 * 512: chunk_seg, per-variable wd / clip, zero padding;
d. a CUDA graph of [pnp_adam_advance, pnp_adam_step] replayed step by step;
e. rejected calls return PNP_ERR_BAD_ARG and leave every buffer untouched;
f. the exact cases and the graph again under PNP_PDL=1, in their own process.

Each real-valued test prints its worst ratio |got - ref| / magnitude next to TAU."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from oracle import optim_exact as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
BAD_ARG = 100001

# (id, optimizer, n, segments, grad_scale, segments with g = 0, monotone chunk_seg).  The CPU file maps each to what it reaches.
EXACT_CASES = [
    ("adam_1chunk", "adam", 1024, 1, 1.0, 0, True),
    ("adam_3chunks_s05", "adam", 3 * 1024, 3, 0.5, 1, False),
    ("adam_300seg_s025", "adam", 1024 * 1024, 300, 0.25, 7, False),
    ("adam_2p24", "adam", 1 << 24, 301, 1.0, 3, False),
    ("rms_1chunk", "rmsprop", 1024, 1, 1.0, 0, True),
    ("rms_3chunks_s025", "rmsprop", 3 * 1024, 3, 0.25, 1, False),
    ("rms_300seg_s05", "rmsprop", 1024 * 1024, 300, 0.5, 7, False),
    ("rms_2p24", "rmsprop", 1 << 24, 301, 1.0, 3, False),
    ("mom_1chunk", "momentum", 1024, 1, 0.5, 0, True),
    ("mom_300seg_s025", "momentum", 1024 * 1024, 300, 0.25, 7, False),
    ("mom_2p24", "momentum", 1 << 24, 301, 1.0, 3, False),
]
ARENA_SIZES = [1, 1023, 1024, 1025, 3 * 3 * 512 * 512]


def _lib():
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C, runtime as rt
    return _C, rt


def ptr(t):
    return None if t is None else t.data_ptr()


def dev(c):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in c.items()}


def launch(_C, rt, kind, d, lr_t=None, state_t=None, seg_clip="case", checked=True):
    """one step of `kind` on the device case d (updated in place); returns the launcher's code"""
    if kind == "adam":
        args = ("pnp_adam_step", ptr(d["theta"]), ptr(d["grad"]), ptr(d["m"]), ptr(d["v"]), d["n"], ptr(d["chunk_seg"]),
                ptr(d["seg_wd"]), ptr(state_t), d["b1"], d["b2"], d["eps"], d["grad_scale"], rt.stream())
    elif kind == "rmsprop":
        clip = d.get("seg_clip") if seg_clip == "case" else seg_clip
        args = ("pnp_rmsprop_step", ptr(d["theta"]), ptr(d["grad"]), ptr(d["ms"]), ptr(d["mom"]), d["n"], ptr(d["chunk_seg"]),
                ptr(d["seg_wd"]), ptr(clip), ptr(lr_t), d["decay"], d["momentum"], d["eps"], d["grad_scale"], rt.stream())
    else:
        args = ("pnp_momentum_step", ptr(d["theta"]), ptr(d["grad"]), ptr(d["accum"]), d["n"], ptr(d["chunk_seg"]), ptr(d["seg_wd"]),
                ptr(lr_t), d["momentum"], d["grad_scale"], rt.stream())
    if checked:
        _C.call(*args)
        return 0
    return getattr(_C.lib, args[0])(*args[1:])


def scalars(kind, c):
    """(lr_t, state_t) device scalars of a case"""
    if kind == "adam":
        return None, torch.tensor(c["state"], dtype=torch.float64, device=DEV)
    return torch.tensor([c["lr"]], dtype=torch.float32, device=DEV), None


def run_exact(kind, c, tag, with_clip=True):
    _C, rt = _lib()
    cc = dict(c) if with_clip else {k: v for k, v in c.items() if k != "seg_clip"}
    ref = O.reference(kind, cc)
    outs = O.OUTPUTS[kind]
    assert O.fp32_exact(*ref["inter"], *[ref[k] for k in outs]), "%s: an intermediate is not an fp32 value" % tag
    d = dev(cc)
    lr_t, state_t = scalars(kind, cc)
    launch(_C, rt, kind, d, lr_t, state_t, seg_clip=d.get("seg_clip"))
    torch.cuda.synchronize()
    for k in outs:
        got = d[k].cpu()
        if not torch.equal(got.double(), ref[k]):
            bad = (got.double() != ref[k]).nonzero().flatten()
            i = int(bad[0])
            raise AssertionError("%s: %s differs at %d of %d elements, first %d: got %r want %r" % (
                tag, k, bad.numel(), got.numel(), i, float(got[i]), float(ref[k][i])))
    return ref


@pytest.mark.parametrize("case", EXACT_CASES, ids=[c[0] for c in EXACT_CASES])
def test_step_exact(case):
    tag, kind, n, nseg, gscale, zero_g, mono = case
    c = O.dyadic_case(kind, n, nseg, gscale, seed=n % 1000 + nseg, zero_g_segments=zero_g, monotone=mono)
    run_exact(kind, c, tag)
    if kind == "rmsprop":
        clip = O.per_element(c["seg_clip"], c["chunk_seg"]).float()
        assert bool(c["edge"].any()), tag + ": no element sits on the clip edge"
        run_exact(kind, c, tag + " seg_clip NULL", with_clip=False)
        # the case must clip somewhere, and leave theta beyond |clip| untouched where clip = 0
        ref = O.reference(kind, c)
        assert bool(((ref["theta"].abs() == clip.double()) & (clip > 0)).any()), tag + ": nothing lands on +-clip"


def test_adam_advance_matches_double():
    """state after t = 1 .. 50 advances equals the Python double computation bit for bit (betas promoted from fp32)"""
    _C, rt = _lib()
    for b1, b2, lr in ((0.9, 0.999, 1e-3), (0.5, 0.75, 2e-4), (0.99, 0.9999, 0.1)):
        st = [1.0, 1.0, lr, 0.0]
        state_t = torch.tensor(st, dtype=torch.float64, device=DEV)
        for t in range(1, 51):
            _C.call("pnp_adam_advance", ptr(state_t), b1, b2, rt.stream())
            st = O.adam_advance(st, b1, b2)
            got = state_t.tolist()
            assert got == st, "b1 %g b2 %g t %d: state %r, want %r" % (b1, b2, t, got, st)


# ------------------------------------------------------------------------------------------------
# b. real-valued
# ------------------------------------------------------------------------------------------------
def real_case(kind, momentum, seed, n=64 * 1024, nseg=40):
    """randn theta, g, first moments; second moments of the order of g^2; wd in [1e-3, 1e-1], so that wd |theta| >> 1e-3 |g|.
    A quarter of the segments are tiny: g ~ 1e-9, wd ~ 1e-9, theta ~ 1e-3, so that their second moment is of the order of eps
    and the place of eps matters"""
    gen = torch.Generator().manual_seed(seed)
    chunk_seg = O.segment_table(n // 1024, nseg, gen)
    tiny_seg = torch.rand(nseg, generator=gen) < 0.25
    seg_wd = (10 ** (-1 - 2 * torch.rand(nseg, generator=gen)) * torch.where(tiny_seg, 1e-8, 1.0)).float()
    tiny = O.per_element(tiny_seg.float(), chunk_seg) > 0
    scale = torch.where(tiny, 1e-9, 1e-3).float()
    theta = torch.randn(n, generator=gen) * torch.where(tiny, 1e-3, 1.0).float()
    grad = torch.randn(n, generator=gen) * scale
    sec = (torch.randn(n, generator=gen) * scale) ** 2 + (scale * 0.1) ** 2
    first = torch.randn(n, generator=gen) * scale
    c = dict(chunk_seg=chunk_seg, seg_wd=seg_wd, grad_scale=0.5, n=n, theta=theta, grad=grad)
    if kind == "adam":
        c.update(m=first, v=sec, state=O.adam_advance(O.adam_advance([0.9 ** 5, 0.999 ** 5, 1e-3, 0.0], 0.9, 0.999), 0.9, 0.999),
                 b1=0.9, b2=0.999, eps=1e-8)
    elif kind == "rmsprop":
        c.update(ms=sec, mom=first * float(momentum > 0), lr=3e-4, decay=0.9, momentum=momentum,
                 eps=1e-10, seg_clip=torch.where(torch.rand(nseg, generator=gen) < 0.5, 0.0, 0.5).float())
    else:
        c.update(accum=first, lr=0.2, momentum=0.2)
    return c


REAL = [("adam", 0.0), ("rmsprop", 0.0), ("rmsprop", 0.9), ("momentum", 0.2)]


@pytest.mark.parametrize("kind,momentum", REAL, ids=["adam", "rmsprop_mom0", "rmsprop_mom09", "momentum"])
def test_step_real(kind, momentum):
    """five steps from a randn state; each compared per element with the reference from the kernel's own previous state"""
    _C, rt = _lib()
    c = real_case(kind, momentum, seed=17)
    d = dev(c)
    worst = 0.0
    for step in range(5):
        if kind == "adam":
            c["state"] = O.adam_advance(c["state"], c["b1"], c["b2"])
            d["state"] = c["state"]
        lr_t, state_t = scalars(kind, c)
        ref = O.reference(kind, c)
        launch(_C, rt, kind, d, lr_t, state_t)
        torch.cuda.synchronize()
        for k in O.OUTPUTS[kind]:
            got = d[k].cpu()
            mag = ref[O.MAGS[k]]
            ratio = O.worst_ratio(got, ref[k], mag)
            worst = max(worst, ratio)
            assert bool(((got.double() - ref[k]).abs() <= O.gamma() * mag).all()), \
                "%s step %d %s: beyond the first-order gamma_%d bound (ratio %.3e)" % (kind, step, k, O.GAMMA_K, ratio)
            bad = int(((got.double() - ref[k]).abs() > O.TAU[kind] * mag).sum())
            assert bad == 0, "%s step %d %s: %d elements beyond tau %.3e (worst ratio %.3e)" % (kind, step, k, bad, O.TAU[kind], ratio)
            c[k] = got
    print("  RATIO %-9s momentum %-4g worst |got-ref|/magnitude %.3e  tau %.3e  gamma_%d %.3e" % (
        kind, momentum, worst, O.TAU[kind], O.GAMMA_K, O.gamma()))


# ------------------------------------------------------------------------------------------------
# c. through optim.Arena
# ------------------------------------------------------------------------------------------------
def test_arena_segments_padding_and_per_variable_hyper_parameters():
    _C, rt = _lib()
    from pnp_b200 import optim
    gen = torch.Generator().manual_seed(3)
    vs = [(torch.randint(-16, 17, (s,), generator=gen).float() * 0.25).to(DEV) for s in ARENA_SIZES]
    arena = optim.Arena(vs)
    want_seg = sum(([i] * -(-s // 1024) for i, s in enumerate(ARENA_SIZES)), [])
    assert arena.chunk_seg.tolist() == want_seg
    wd = [0.0, 0.25, 0.5, 0.75, 0.125]
    clip = [2.0, 0.0, 1.5, 2.5, 3.0]
    opt = optim.RMSProp(arena, lr=0.125, decay=0.5, momentum=0.5, eps=0.0, weight_decay=wd, clip=clip)
    for step in range(3):
        for v in vs:      # fresh dyadic theta / g / mom each step, so that every intermediate stays an fp32 value
            v.copy_((torch.randint(-16, 17, v.shape, generator=gen).float() * 0.25).to(DEV))
            v.grad.copy_((torch.randint(-8, 9, v.shape, generator=gen).float()).to(DEV))
        opt.mom.zero_()
        for o, n in arena.offsets:        # the padding's momentum stays 0, as the optimizer leaves it
            opt.mom[o:o + n] = (torch.randint(-128, 129, (n,), generator=gen).float() / 16).to(DEV)
        # the expected per-chunk tables from the variable list itself, not from the arena's
        wd_chunk = torch.tensor(sum(([w] * -(-s // 1024) for s, w in zip(ARENA_SIZES, wd)), []))
        clip_chunk = torch.tensor(sum(([c] * -(-s // 1024) for s, c in zip(ARENA_SIZES, clip)), []))
        th, g, mom = arena.theta.cpu(), arena.grad.cpu(), opt.mom.cpu()
        gg = wd_chunk.double().repeat_interleave(1024) * th.double() + g.double()
        opt.ms.copy_((2.0 * 4.0 ** 4 - gg ** 2).float().to(DEV))     # the new ms is 256: sqrt exact
        ms = opt.ms.cpu()
        ident = torch.arange(th.numel() // 1024, dtype=torch.int32)
        ref = O.rmsprop_step(th, g, ms, mom, ident, wd_chunk.float(), clip_chunk.float(), 0.125, 0.5, 0.5, 0.0, 1.0)
        assert O.fp32_exact(*ref["inter"], ref["theta"])
        opt.step()
        torch.cuda.synchronize()
        assert torch.equal(arena.theta.cpu().double(), ref["theta"]), "step %d: theta" % step
        assert torch.equal(opt.ms.cpu().double(), ref["ms"]) and torch.equal(opt.mom.cpu().double(), ref["mom"]), "step %d" % step
        for (o, n), s in zip(arena.offsets, ARENA_SIZES):
            pad = arena.theta[o + n: o + -(-s // 1024) * 1024]
            assert bool((pad == 0).all()), "step %d: padding of the %d-element variable moved" % (step, s)


# ------------------------------------------------------------------------------------------------
# d. captured graph
# ------------------------------------------------------------------------------------------------
def test_adam_graph_reads_the_advanced_lr():
    """[pnp_adam_advance, pnp_adam_step] captured once and replayed: after each replay the state equals the Python advance
    bit for bit and theta / m / v equal the reference step with that state's lr_t, within TAU"""
    _C, rt = _lib()
    c = real_case("adam", 0.0, seed=29, n=8 * 1024, nseg=5)
    c["state"] = [1.0, 1.0, 1e-3, 0.0]
    d = dev(c)
    state_t = torch.tensor(c["state"], dtype=torch.float64, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            _C.call("pnp_adam_advance", ptr(state_t), c["b1"], c["b2"], torch.cuda.current_stream().cuda_stream)
            _C.call("pnp_adam_step", ptr(d["theta"]), ptr(d["grad"]), ptr(d["m"]), ptr(d["v"]), d["n"], ptr(d["chunk_seg"]),
                    ptr(d["seg_wd"]), ptr(state_t), c["b1"], c["b2"], c["eps"], c["grad_scale"], torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert state_t.tolist() == [1.0, 1.0, 1e-3, 0.0], "capture must not run the kernels"
    for t in range(1, 4):
        prev = c["state"]
        c["state"] = O.adam_advance(prev, c["b1"], c["b2"])
        ref = O.reference("adam", c)
        stale = O.reference("adam", c, state=prev)
        graph.replay()
        torch.cuda.synchronize()
        assert state_t.tolist() == c["state"], "replay %d: state %r want %r" % (t, state_t.tolist(), c["state"])
        for k in ("theta", "m", "v"):
            got = d[k].cpu()
            ratio = O.worst_ratio(got, ref[k], ref[O.MAGS[k]])
            assert ratio <= O.TAU["adam"], "replay %d %s: ratio %.3e beyond tau" % (t, k, ratio)
            c[k] = got
        assert O.worst_ratio(c["theta"], stale["theta"], ref["mag_theta"]) > 100 * O.TAU["adam"], "lr_t does not matter here"
    del graph


# ------------------------------------------------------------------------------------------------
# e. rejected calls
# ------------------------------------------------------------------------------------------------
REJECT = [(kind, what, change) for kind in ("adam", "rmsprop", "momentum") for what, change in
          [("n_not_multiple", {"n": 1000}), ("n_zero", {"n": 0}), ("n_negative", {"n": -1024})] +
          [("null_" + k, {k: None}) for k in O.OUTPUTS[kind] + ("grad", "chunk_seg", "seg_wd", "scalar")]]


@pytest.mark.parametrize("kind,what,change", REJECT, ids=["%s_%s" % r[:2] for r in REJECT])
def test_rejected_calls_leave_buffers_untouched(kind, what, change):
    _C, rt = _lib()
    key = next(iter(change))
    c = O.dyadic_case(kind, 2048, 2, 1.0, seed=5)
    d = dev(c)
    before = {k: d[k].clone() for k in O.OUTPUTS[kind]}
    lr_t, state_t = scalars(kind, c)
    if key == "scalar":
        lr_t, state_t = None, None
    else:
        d.update(change)
    torch.cuda.synchronize()
    rc = launch(_C, rt, kind, d, lr_t, state_t, checked=False)
    torch.cuda.synchronize()
    assert rc == BAD_ARG, "%s %s: returned %d" % (kind, what, rc)
    for k, b in before.items():
        if d[k] is not None:
            assert torch.equal(d[k], b), "%s %s: %s changed" % (kind, what, k)


# ------------------------------------------------------------------------------------------------
# f. PDL
# ------------------------------------------------------------------------------------------------
@pytest.mark.timeout(300)
def test_exact_cases_under_pdl():
    """programmatic dependent launch lets each kernel start before its predecessor ends: the step must still see the advanced
    state and the previous step's outputs"""
    env = dict(os.environ, PNP_PDL="1")
    code = ("import sys; sys.path.insert(0, %r); from tests import test_optim_exact_gpu as T; "
            "[T.test_step_exact(c) for c in T.EXACT_CASES if '2p24' not in c[0]]; T.test_adam_advance_matches_double(); "
            "T.test_adam_graph_reads_the_advanced_lr(); print('pdl ok')" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=280)
    assert r.returncode == 0 and "pdl ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
