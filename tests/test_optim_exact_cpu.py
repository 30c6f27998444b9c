"""The optimizer references (oracle/optim_exact.py) without a GPU: the exact cases of tests/test_optim_exact_gpu.py meet their
precondition and reach what they claim, the references follow the update rules, pnp_adam_advance's double state, and negative
controls: each realistic bug of a step breaks the exact cases or exceeds TAU by a wide margin, which is printed."""
import math

import pytest
import torch

from oracle import optim_exact as O
from tests.test_optim_exact_gpu import ARENA_SIZES, EXACT_CASES, REAL, REJECT, real_case

SMALL = [c for c in EXACT_CASES if c[2] <= 1024 * 1024]      # the 2^24 cases take gigabytes of fp64 temporaries on the CPU

# what each GPU case reaches: entry point and path
CASE_MAP = {
    "adam_1chunk": ("pnp_adam_step", "one CTA, one segment"),
    "adam_3chunks_s05": ("pnp_adam_step", "3 CTAs, a g = 0 segment, grad_scale 0.5"),
    "adam_300seg_s025": ("pnp_adam_step", "1024 CTAs, 300 non-monotone segments, grad_scale 0.25"),
    "adam_2p24": ("pnp_adam_step", "16384 CTAs, 301 segments"),
    "rms_1chunk": ("pnp_rmsprop_step", "one CTA, theta on and beyond +-clip, seg_clip and NULL"),
    "rms_3chunks_s025": ("pnp_rmsprop_step", "clip = 0 and clip > 0 segments, grad_scale 0.25"),
    "rms_300seg_s05": ("pnp_rmsprop_step", "300 non-monotone segments, grad_scale 0.5"),
    "rms_2p24": ("pnp_rmsprop_step", "16384 CTAs"),
    "mom_1chunk": ("pnp_momentum_step", "one CTA, grad_scale 0.5"),
    "mom_300seg_s025": ("pnp_momentum_step", "300 non-monotone segments"),
    "mom_2p24": ("pnp_momentum_step", "16384 CTAs"),
}


def _case(c):
    tag, kind, n, nseg, gscale, zero_g, mono = c
    return kind, O.dyadic_case(kind, n, nseg, gscale, seed=n % 1000 + nseg, zero_g_segments=zero_g, monotone=mono)


def test_case_table():
    assert {c[0] for c in EXACT_CASES} == set(CASE_MAP)
    assert {v[0] for v in CASE_MAP.values()} == {"pnp_adam_step", "pnp_rmsprop_step", "pnp_momentum_step"}
    assert {c[4] for c in EXACT_CASES} == {1.0, 0.5, 0.25}
    assert {1024, 3 * 1024, 1 << 24} <= {c[2] for c in EXACT_CASES}
    assert {k for k, _, _ in REJECT} == {"adam", "rmsprop", "momentum"}
    assert {1, 1023, 1024, 1025} <= set(ARENA_SIZES)


@pytest.mark.parametrize("case", SMALL, ids=[c[0] for c in SMALL])
def test_exact_case_preconditions(case):
    kind, c = _case(case)
    ref = O.reference(kind, c)
    assert O.fp32_exact(*ref["inter"], *[ref[k] for k in O.OUTPUTS[kind]])
    seg = c["chunk_seg"].long()
    if case[3] >= 300:
        assert bool((seg[1:] < seg[:-1]).any()) and seg.unique().numel() < seg.numel(), "non-monotone with repeats"
    if case[5]:
        gz = (c["grad"].view(-1, 1024) == 0).all(1)
        assert bool(gz.any()), "a segment with g = 0"
    if kind == "rmsprop":
        clip = O.per_element(c["seg_clip"], c["chunk_seg"])
        assert bool(c["edge"].any()) and bool(((ref["theta"].abs() == clip) & (clip > 0)).any())
        assert bool((clip == 0).any()) or case[3] == 1


def test_references_follow_the_update_rules():
    """one element by hand: the references against the textbook formulas"""
    one = torch.zeros(1024, dtype=torch.int32)[:1]
    th, g = torch.full((1024,), 0.5), torch.full((1024,), -2.0)
    wd = torch.tensor([0.25])
    gg = 0.25 * 0.5 + -2.0 * 0.5
    r = O.adam_step(th, g, torch.full((1024,), 0.125), torch.full((1024,), 4.0), one, wd, [0.25, 0.0625, 0.1, 0.0625], 0.5, 0.5, 0.0, 0.5)
    m, v = 0.5 * 0.125 + 0.5 * gg, 0.5 * 4.0 + 0.5 * gg * gg
    assert float(r["m"][0]) == m and float(r["v"][0]) == v and float(r["theta"][0]) == 0.5 - 0.0625 * m / math.sqrt(v)
    r = O.rmsprop_step(th, g, torch.full((1024,), 4.0), torch.full((1024,), 0.25), one, wd, torch.tensor([0.375]), 0.125, 0.5, 0.5, 0.0,
                       0.5)
    ms = 0.5 * 4.0 + 0.5 * gg * gg
    mo = 0.5 * 0.25 + 0.125 * gg / math.sqrt(ms)
    assert float(r["ms"][0]) == ms and float(r["mom"][0]) == mo and float(r["theta"][0]) == min(max(0.5 - mo, -0.375), 0.375)
    r = O.momentum_step(th, g, torch.full((1024,), 0.25), one, wd, 0.125, 0.5, 0.5)
    assert float(r["accum"][0]) == 0.5 * 0.25 + gg and float(r["theta"][0]) == 0.5 - 0.125 * (0.125 + gg)


def test_adam_advance_promotes_fp32_betas():
    st = [1.0, 1.0, 1e-3, 0.0]
    for t in range(1, 51):
        st = O.adam_advance(st, 0.9, 0.999)
        b1, b2 = O.f32(0.9), O.f32(0.999)
        assert st[0] == b1 ** t or abs(st[0] - b1 ** t) <= 64 * 2.0 ** -53 * st[0]
        assert st[3] == 1e-3 * math.sqrt(1.0 - st[1]) / (1.0 - st[0])
    assert O.f32(0.9) != 0.9 and st[0] != 0.9 ** 50


# ------------------------------------------------------------------------------------------------
# negative controls
# ------------------------------------------------------------------------------------------------
def _diff(kind, ref, mut):
    return sum(int((ref[k] != mut[k]).sum()) for k in O.OUTPUTS[kind] if k in mut)


def _clamp(t, clip):
    return torch.where(clip > 0, torch.minimum(torch.maximum(t, -clip), clip), t)


def exact_mutant(kind, c, mutation):
    """the step with one bug, on an exact case; None where the bug does not apply to `kind`"""
    n, nch = c["n"], c["n"] // 1024
    if mutation == "wd_ignored":
        return O.reference(kind, c, seg_wd=torch.zeros_like(c["seg_wd"]))
    if mutation == "wd_by_block_index":
        pad = torch.cat([c["seg_wd"], torch.zeros(max(0, nch - c["seg_wd"].numel()))])
        return O.reference(kind, c, chunk_seg=torch.arange(nch, dtype=torch.int32), seg_wd=pad,
                           **({"seg_clip": torch.cat([c["seg_clip"], torch.zeros(max(0, nch - c["seg_clip"].numel()))])[
                               c["chunk_seg"].long()]} if kind == "rmsprop" else {}))
    if mutation == "grad_scale_on_wd":
        return O.reference(kind, c, seg_wd=c["seg_wd"] * c["grad_scale"])
    if mutation == "clip_when_zero" and kind == "rmsprop":
        r = O.reference(kind, c)
        clip = O.per_element(c["seg_clip"], c["chunk_seg"], n)
        return dict(r, theta=torch.where(clip == 0, torch.zeros_like(r["theta"]), r["theta"]))
    if mutation == "clip_before_update" and kind == "rmsprop":
        r = O.reference(kind, c)
        clip = O.per_element(c["seg_clip"], c["chunk_seg"], n)
        return dict(r, theta=_clamp(c["theta"].double(), clip) - r["mom"])
    if mutation == "lr_for_lr_t" and kind == "adam":
        st = list(c["state"])
        return O.reference(kind, c, state=st[:3] + [st[2]])
    return None


EXACT_MUTATIONS = ["wd_ignored", "wd_by_block_index", "grad_scale_on_wd", "clip_when_zero", "clip_before_update", "lr_for_lr_t"]


@pytest.mark.parametrize("mutation", EXACT_MUTATIONS)
def test_exact_cases_reject(mutation):
    total, hit = 0, []
    for case in SMALL:
        kind, c = _case(case)
        mut = exact_mutant(kind, c, mutation)
        if mut is None:
            continue
        d = _diff(kind, O.reference(kind, c), mut)
        total += d
        if d:
            hit.append(case[0])
    print("  %-20s changes %8d output elements, in cases %s" % (mutation, total, hit))
    assert total > 0


def real_mutant(kind, c, mutation):
    """one step with one bug on a real-valued case"""
    if mutation == "adam_eps_inside_sqrt" and kind == "adam":
        r = O.reference(kind, c)
        upd = O.f32(c["state"][3]) * r["m"] / (r["v"] + O.f32(c["eps"])).sqrt()
        return dict(r, theta=c["theta"].double() - upd)
    if mutation == "rmsprop_eps_outside_sqrt" and kind == "rmsprop":
        r = O.reference(kind, c)
        wd = O.per_element(c["seg_wd"], c["chunk_seg"], c["n"])
        gg = wd * c["theta"].double() + c["grad"].double() * c["grad_scale"]
        mom = O.f32(c["momentum"]) * c["mom"].double() + O.f32(c["lr"]) * gg / (r["ms"].sqrt() + O.f32(c["eps"]))
        clip = O.per_element(c["seg_clip"], c["chunk_seg"], c["n"])
        return dict(r, mom=mom, theta=_clamp(c["theta"].double() - mom, clip))
    if mutation == "advance_one_behind" and kind == "adam":
        behind = c["state"]                    # the state before the advance this step should have read
        return O.reference(kind, c, state=behind)
    if mutation == "wd_ignored":
        return O.reference(kind, c, seg_wd=torch.zeros_like(c["seg_wd"]))
    return None


REAL_MUTATIONS = ["adam_eps_inside_sqrt", "rmsprop_eps_outside_sqrt", "advance_one_behind", "wd_ignored"]


@pytest.mark.parametrize("mutation", REAL_MUTATIONS)
def test_real_cases_reject(mutation):
    """the worst ratio |mutant - ref| / magnitude over the GPU file's real-valued cases, as a multiple of TAU"""
    worst = 0.0
    for kind, momentum in REAL:
        c = real_case(kind, momentum, seed=17)
        if kind == "adam":
            prev = c["state"]
            c["state"] = O.adam_advance(prev, c["b1"], c["b2"])
        mut = real_mutant(kind, dict(c, state=prev) if mutation == "advance_one_behind" and kind == "adam" else c, mutation)
        if mut is None:
            continue
        ref = O.reference(kind, c)
        for k in O.OUTPUTS[kind]:
            if k in mut:
                worst = max(worst, O.worst_ratio(mut[k].float(), ref[k], ref[O.MAGS[k]]) / O.TAU[kind])
    print("  %-26s worst ratio %.3g x tau" % (mutation, worst))
    assert worst > 100


def test_advance_one_behind_changes_every_lr_t():
    st, prev = [1.0, 1.0, 1e-3, 0.0], None
    for t in range(1, 51):
        prev, st = st, O.adam_advance(st, 0.9, 0.999)
        assert abs(st[3] - prev[3]) > 1e-4 * st[3], t


def test_tau_values_are_calibrated():
    """TAU sits well inside the first-order rigorous bound and well above one fp32 rounding"""
    for k, tau in O.TAU.items():
        assert O.U32 < tau < O.gamma(), (k, tau)
