"""oracle/node_exact.py against fp64 autograd of the same node built from oracle/tf14_torch.py, and the tables it derives from
the reference trace against the reference's own numbers.  The references must agree with autograd to 1e-12 (relative to the
largest value), and the two negative controls of tests/test_node_taps_gpu.py that a gradient ledger cannot see must move the
reference's answer by more than its bound."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import layer_exact as LX
from oracle import node_exact as N
from oracle import tf14_torch as T

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1e-12


def _trace():
    with open(os.path.join(HERE, "golden", "reference_graph_trace.json")) as f:
        return json.load(f)


def _close(got, ref):
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    scale = max(1.0, float(ref.abs().max()))
    err = float((got - ref).abs().max())
    assert err <= TOL * scale, err


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(shape, seed):
    return torch.randn(shape, generator=_gen(seed), dtype=torch.float64)


def test_maxpool_against_autograd():
    x = _randn((2, 6, 8, 5), 1).requires_grad_()
    y = T.max_pool2d(x)
    dy = _randn(tuple(y.shape), 2)
    y.backward(dy)
    assert torch.equal(N.maxpool_fwd(x.detach()), y.detach())
    assert torch.equal(N.maxpool_bwd(x.detach(), dy), x.grad)


def test_maxpool_backward_routes_to_the_first_maximum():
    x = torch.zeros(1, 2, 2, 1, dtype=torch.float64)          # a window of four equal values
    got = N.maxpool_bwd(x, torch.ones(1, 1, 1, 1, dtype=torch.float64))
    assert got.reshape(-1).tolist() == [1.0, 0.0, 0.0, 0.0]


@pytest.mark.parametrize("B", [1, 2])
def test_disc_input_against_autograd(B):
    """[PS(c4) x3 | PS(c6) | PS(b7) | PS(c9) | logits | argmax] with the group counts of the real graph scaled down (r = 2)"""
    r, a, NC = 2, 3, 5
    Gs = (2, 1, 3, 1)
    srcs = [_randn((B, a, a, G * r * r), 10 + i).requires_grad_() for i, G in enumerate(Gs)]
    logits = _randn((B, a * r, a * r, NC), 20).requires_grad_()
    parts = [T.PS(s, r, G, B).repeat(1, 1, 1, t) for s, G, t in zip(srcs, Gs, N.DISC_NTILES)]
    am = logits.detach().argmax(-1, keepdim=True).double()
    out = torch.cat(parts + [logits, am], dim=3)
    order_b1 = 1 if B == 1 else 0
    assert torch.equal(N.disc_input_fwd([s.detach() for s in srcs], logits.detach(), r, order_b1), out.detach())
    dout = _randn(tuple(out.shape), 30)
    out.backward(dout)
    coff = 0
    for s, G, t in zip(srcs, Gs, N.DISC_NTILES):
        _close(N.disc_input_bwd(dout, r, G, coff, t, order_b1), s.grad)
        coff += G * t
    _close(N.channel_slice(dout, dout.shape[-1], coff, NC).reshape(logits.shape), logits.grad)


def test_fc_against_autograd():
    B, F = 4, 300
    x = _randn((B, F), 40).requires_grad_()
    w = _randn((F, 1), 41).requires_grad_()
    out = x @ w
    dout = _randn((B, 1), 42)
    out.backward(dout)
    ref, bound = N.fc_fwd(x.detach(), w.detach())
    _close(ref, out.detach())
    assert float(bound.min()) > 0
    _close(N.fc_dx(dout, w.detach())[0], x.grad)
    before = _randn((F, 1), 43)
    _close(N.fc_dw(x.detach(), dout, before)[0] - before, w.grad)


def test_mean_combo_against_autograd():
    n = 6
    a, b = _randn((n, 1), 50).requires_grad_(), _randn((n, 1), 51).requires_grad_()
    ca, cb = N.f32(-0.002), N.f32(0.002)
    out = ca * a.mean() + cb * b.mean()
    out.backward(torch.tensor(0.3, dtype=torch.float64))
    _close(N.mean_combo_fwd(a.detach(), ca, b.detach(), cb)[0], out.detach())
    _close(N.mean_combo_fwd(a.detach(), ca)[0], ca * a.detach().mean())
    _close(N.mean_combo_bwd(0.3, ca, n, (n, 1))[0], a.grad)
    _close(N.mean_combo_bwd(0.3, cb, n, (n, 1))[0], b.grad)


def test_segloss_against_autograd():
    B, H, C = 2, 6, 5
    logits = (3 * _randn((B, H, H, C), 60)).requires_grad_()
    y = torch.nn.functional.one_hot(torch.randint(0, C, (B, H, H), generator=_gen(61)), C).double()
    wce, dice = T.softmax_weighted_loss(logits, y), T.dice_loss(logits, y)
    g_wce, g_dice = 0.7, -1.3
    torch.autograd.backward([wce, dice], [torch.tensor(g_wce, dtype=torch.float64), torch.tensor(g_dice, dtype=torch.float64)])
    P = B * H * H
    acc, acc_bound = N.segloss_acc(logits.detach(), y)
    (out, _), (coef, _) = N.segloss_out(acc, P, C)
    _close(out, torch.stack([wce.detach(), dice.detach()]))
    _close(N.segloss_bwd(logits.detach(), y, coef, g_wce, g_dice)[0], logits.grad)
    assert float(acc_bound.min()) > 0


def test_l2_sum_against_autograd():
    ws = [_randn((3, 3, 4, 8), 70).requires_grad_(), _randn((12,), 71).requires_grad_()]
    total = 2 * T.l2_loss(ws[0]) + T.l2_loss(ws[1])
    total.backward()
    ref, bound = N.l2_sum([w.detach() for w in ws], [2, 1])
    assert abs(ref - float(total.detach())) <= TOL * float(total.detach()) and 0 < bound < 1e-5 * ref
    _close(ws[0].grad, 2 * ws[0].detach())


def test_ledger_against_autograd():
    """one tensor consumed by three nodes: autograd's gradient is the sum of what their backwards return"""
    x = _randn((2, 4, 4, 3), 80).requires_grad_()
    h = x * 1.0
    uses = [T.max_pool2d(h).sum(), T.l2_loss(h), (h.reshape(2, -1) @ _randn((48, 1), 81)).sum()]
    parts = [torch.autograd.grad(u, h, retain_graph=True)[0] for u in uses]
    torch.autograd.backward(uses)
    ref, bound = N.ledger(parts)
    _close(ref, x.grad)
    assert float(bound.max()) > 0 and float(N.ledger(parts[:1])[1].max()) == 0.0


def test_two_tiles_of_c4_are_rejected_by_the_disc_input_backward():
    """negative control 1: the backward adds two of c4's three tiles; the stage is exact, so any change is a rejection"""
    dout = torch.randn((2, 8, 8, 12), generator=_gen(90))
    good = N.disc_input_bwd(dout, 2, 2, 0, 3, 0)
    bad = N.disc_input_bwd(dout, 2, 2, 0, 3, 0, tiles=2)
    assert not torch.equal(good, bad)


def test_an_overwriting_fc_dw_is_rejected():
    """negative control 2: the second critic call zeroes dw before its own chain, so the slot holds the second sum only"""
    B, F = 4, 256
    xs = [torch.randn((B, F), generator=_gen(91 + i)) for i in range(2)]
    ds = [torch.randn((B, 1), generator=_gen(93 + i)) for i in range(2)]
    first, _ = N.fc_dw(xs[0], ds[0])
    ref, bound = N.fc_dw(xs[1], ds[1], first.float())
    overwritten = N.fc_dw(xs[1], ds[1])[0]
    assert LX.ratio(overwritten, ref, bound) > 1


def test_regularisers_from_the_weight_lists_equal_the_reference():
    """the multiplicities of the recorded weight lists reproduce adversarial.py's dis_reg / gen_reg / fixed_coeff_reg from its
    own l2 values"""
    tr = _trace()
    c = tr["cost_numeric"]
    for case in c["cases"]:
        ck = case["cost_kwargs"]
        lam = ck.get("lambda_mask_loss", 1.0)
        got = N.regularisers(tr, ck, lam, lambda n: c["l2"][n])
        for key, v in got.items():
            assert v == pytest.approx(case[key], rel=1e-12), (key, lam)


@pytest.mark.parametrize("dis_sub_iter,gen_sub_iter", [(1, 1), (20, 3)])
def test_weight_decay_is_the_gradient_of_the_regularisers(dis_sub_iter, gen_sub_iter):
    """wd * w = d(dis_reg / dis_sub_iter) / dw and d(gen_reg / gen_sub_iter) / dw, by fp64 autograd of the l2 terms; the segmenter's
    regularizer_loss likewise"""
    tr = _trace()
    ck = {"gan_regularizer": 1e-4, "miu_dis": 0.002, "miu_gen": 0.002, "regularizer": 1e-4}
    lam = 0.3
    names = sorted(set(sum(tr["weight_lists"].values(), [])) | set(tr["source_segmenter"]["conv_weights"]))
    w = {n: _randn((3,), 100 + i).requires_grad_() for i, n in enumerate(names)}
    l2 = lambda n: T.l2_loss(w[n])  # noqa: E731
    reg = N.regularisers(tr, ck, lam, l2)
    wd_d, wd_g = N.gan_weight_decay(tr, ck, lam, dis_sub_iter, gen_sub_iter)
    for key, wd, div in (("dis_reg", wd_d, dis_sub_iter), ("gen_reg", wd_g, gen_sub_iter)):
        grads = torch.autograd.grad(reg[key] / div, [w[n] for n in names], allow_unused=True)
        for n, g in zip(names, grads):
            want = wd.get(n, 0.0) * w[n].detach()
            _close(torch.zeros(3, dtype=torch.float64) if g is None else g, want)
    wd_s = N.segmenter_weight_decay(tr, ck)
    grads = torch.autograd.grad(N.segmenter_regulariser(tr, ck, l2), [w[n] for n in names], allow_unused=True)
    for n, g in zip(names, grads):
        _close(torch.zeros(3, dtype=torch.float64) if g is None else g, wd_s.get(n, 0.0) * w[n].detach())
    assert max(N.multiplicities(tr["weight_lists"]["cls_weights"]).values()) == 2
    assert max(wd_s.values()) == 2 * ck["regularizer"]           # group_4/Variable_3 is listed twice
    assert tr["optimizer"]["optimizers"][0]["objective"]["dis_reg"] == pytest.approx(1.0 / tr["optimizer"]["train_config_used"]["dis_sub_iter"])


def test_critic_clip_table():
    clip = N.critic_clip(_trace())
    assert len(clip) == 26 and set(clip.values()) == {0.03} and all("Variable" in n for n in clip)
    assert np.isclose(N.f32(0.03), 0.03, rtol=1e-7)


@pytest.mark.parametrize("spread", [3.0, 12.0, 40.0])
def test_segloss_accumulator_bound_covers_an_fp32_evaluation(spread):
    """segloss_reduce_kernel's arithmetic in fp32 (softmax, per-pixel terms, chains of 32 pixels, fp64 above them) stays within
    segloss_acc's bound for logits of any spread"""
    P, C = 4096, 5
    l = (spread * torch.randn((P, C), generator=_gen(120))).float()
    y = torch.nn.functional.one_hot(torch.randint(0, C, (P,), generator=_gen(121)), C).float()
    t = l - l.max(1, keepdim=True).values
    e = torch.exp(t)
    p = e * (1.0 / e.sum(1, keepdim=True))
    terms = torch.cat([y, p * y, p * p, -y * torch.log(p.clamp(0.005, 1.0))], 1)
    got = terms.reshape(P // 32, 32, 4 * C).sum(1).double().sum(0)
    ref, bound = N.segloss_acc(l, y)
    assert LX.ratio(got, ref, bound) <= 1
