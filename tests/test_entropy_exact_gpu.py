"""pnp_entropy_reduce / _finalize / _bwd (elementwise.cu) against oracle/entropy_exact.py at the C-ABI, within the a-priori bound
of DESIGN 6.1 (entropy_exact.bounds, derived from the kernel's expression, not fitted): C of 2, 5 and 8; P of 1, 257 (a partial
CTA), 16 * 256^2 and past the grid cap (a grid-stride sweep); tied logits (H = log C), saturated ones (H = 0, finite
gradients), magnitudes up to 1e4; upstream g of 0, 1 and 3.5; NaN logits; graph-replayed launches against eager ones; every
rejected argument returns PNP_ERR_BAD_ARG and leaves the buffers untouched."""
import math

import numpy as np
import pytest
import torch

from oracle import entropy_exact as E
from tests.cabi import BAD_ARG, DEV, assert_bits, assert_untouched, lib, sentinel, snapshot, sync

pytestmark = pytest.mark.gpu

GRID_CAP_PIXELS = 132 * 64 * 512          # grid_for's cap (PNP_NUM_SMS * 64 CTAs) times the 512 pixels each CTA is sized for


def _launch(_C, rt, x, g):
    """-> (out [1 + C], dlogits) of fp32 logits x [..., C] on the device, upstream g (device scalar)"""
    C = x.shape[-1]
    P = x.numel() // C
    acc = torch.zeros(1 + C, dtype=torch.float64, device=DEV)
    out = sentinel(1 + C)
    dl = sentinel(tuple(x.shape))
    gt = torch.tensor([g], dtype=torch.float32, device=DEV)
    st = rt.stream()
    _C.call("pnp_entropy_reduce", x.data_ptr(), P, C, acc.data_ptr(), st)
    _C.call("pnp_entropy_finalize", acc.data_ptr(), P, C, out.data_ptr(), st)
    _C.call("pnp_entropy_bwd", x.data_ptr(), gt.data_ptr(), dl.data_ptr(), P, C, st)
    sync()
    return out.cpu().double().numpy(), dl.cpu().double().numpy()


def _check(tag, x, g=1.0):
    _C, rt = lib()
    xn = x.cpu().numpy()
    out, dl = _launch(_C, rt, x, g)
    L, pbar, d, _ = E.entropy(xn, g)
    bL, bp, bd = E.bounds(xn, g)
    assert np.all(np.isfinite(out)) and np.all(np.isfinite(dl)), tag
    assert abs(out[0] - L) <= bL, (tag, "loss", out[0], L, bL)
    ep = np.abs(out[1:] - pbar)
    assert np.all(ep <= bp), (tag, "pbar", ep.max(), bp.min())
    ed = np.abs(dl - d)
    i = np.unravel_index(np.argmax(ed - bd), ed.shape)
    assert np.all(ed <= bd), (tag, "dlogits", i, dl[i], d[i], bd[i])
    return out, dl, L, d


def _normal(shape, seed, scale):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=gen, device=DEV) * scale


@pytest.mark.parametrize("C", [2, 5, 8])
@pytest.mark.parametrize("P", [1, 257])
@pytest.mark.parametrize("g", [0.0, 1.0, 3.5])
def test_small_sizes_match_the_oracle(C, P, g):
    _, dl, _, _ = _check("C %d P %d g %g" % (C, P, g), _normal((P, 1, 1, C), 10 * C + P, 3.0), g)
    if g == 0.0:
        assert np.all(dl == 0.0)


@pytest.mark.parametrize("C", [2, 8])
def test_grid_stride_sweep_past_the_grid_cap(C):
    P = GRID_CAP_PIXELS + 12345
    _check("C %d P %d" % (C, P), _normal((1, P, 1, C), 7 + C, 4.0), 1.0)


def test_benchmark_size():
    _check("16 x 256 x 256 x 5", _normal((16, 256, 256, 5), 3, 2.0), 1.0)


@pytest.mark.parametrize("C", [2, 5, 8])
def test_tied_logits_give_log_c(C):
    v = torch.tensor([-1e4, -3.0, 0.0, 0.25, 88.0, 1e4], device=DEV)
    x = v.repeat_interleave(43 * C).reshape(-1, 1, 1, C)          # every pixel's C logits equal
    out, dl, L, _ = _check("tied C %d" % C, x, 1.0)
    assert abs(out[0] - math.log(C)) <= 4 * C * 2.0 ** -24 * math.log(C)
    assert np.all(np.abs(out[1:] - 1.0 / C) <= 4 * 2.0 ** -24)
    assert np.all(np.abs(dl) <= 1e-6 / x.shape[0])


@pytest.mark.parametrize("C", [2, 5, 8])
def test_saturated_logits_give_zero_entropy_and_finite_gradients(C):
    gen = torch.Generator(device=DEV).manual_seed(C)
    P = 1000
    x = torch.rand((P, 1, 1, C), generator=gen, device=DEV) * 50.0 - 25.0
    hot = torch.randint(0, C, (P,), generator=gen, device=DEV)
    gap = 100.0 + torch.rand((P,), generator=gen, device=DEV) * 900.0
    x[torch.arange(P, device=DEV), 0, 0, hot] = x.amax(-1)[:, 0, 0] + gap
    out, dl, _, _ = _check("saturated C %d" % C, x, 3.5)
    assert 0.0 <= out[0] <= 1e-30
    assert np.all(np.isfinite(dl))


@pytest.mark.parametrize("C", [2, 5, 8])
@pytest.mark.parametrize("scale", [1e2, 1e3, 1e4])
def test_large_magnitudes(C, scale):
    gen = torch.Generator(device=DEV).manual_seed(int(scale) + C)
    x = (torch.rand((4, 16, 16, C), generator=gen, device=DEV) * 2.0 - 1.0) * scale
    x[0, 0, 0, :] = scale                                         # ties at the top of the range
    x[0, 0, 1, :] = torch.linspace(scale - 1.0, scale, C, device=DEV)     # near ties, close to |l| = scale
    _check("C %d scale %g" % (C, scale), x, 1.0)


def test_nan_logits_give_a_nan_loss():
    _C, rt = lib()
    for pos in (0, 3):
        x = _normal((2, 8, 8, 5), 5, 2.0)
        x[1, 2, 3, pos] = float("nan")
        out, dl = _launch(_C, rt, x, 1.0)
        assert np.isnan(out[0]) and np.isnan(out[1 + pos]), pos
        assert np.all(np.isnan(dl[1, 2, 3])), pos
        assert np.all(np.isfinite(np.delete(dl.reshape(-1, 5), 64 + 2 * 8 + 3, axis=0)))


def test_graph_replays_equal_eager_launches():
    """the backward reads g from the device on every replay, so replays with a new g equal eager launches bit for bit; the
    loss's fp64 atomic sums may add in another order, which moves the fp32 results by at most one rounding"""
    _C, rt = lib()
    x = _normal((16, 64, 64, 5), 11, 3.0)
    C, P = 5, x.numel() // 5
    acc = torch.zeros(1 + C, dtype=torch.float64, device=DEV)
    out = torch.empty(1 + C, device=DEV)
    dl = torch.empty_like(x)
    gt = torch.tensor([1.0], device=DEV)
    _launch(_C, rt, x, 1.0)                                       # modules loaded before the capture
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            st = rt.stream()
            _C.call("pnp_fill", acc.data_ptr(), 0.0, 2 * (1 + C), st)
            _C.call("pnp_entropy_reduce", x.data_ptr(), P, C, acc.data_ptr(), st)
            _C.call("pnp_entropy_finalize", acc.data_ptr(), P, C, out.data_ptr(), st)
            _C.call("pnp_entropy_bwd", x.data_ptr(), gt.data_ptr(), dl.data_ptr(), P, C, st)
    torch.cuda.current_stream().wait_stream(side)
    for g in (1.0, 3.5, 0.0, 1.0):
        gt.fill_(g)
        graph.replay()
        sync()
        ref_out, ref_dl = _launch(_C, rt, x, g)
        assert_bits("dlogits g %g" % g, dl, torch.from_numpy(ref_dl).float().to(DEV))
        assert np.all(np.abs(out.cpu().double().numpy() - ref_out) <= 2.0 ** -23 * np.abs(ref_out)), g


def test_rejected_arguments():
    _C, rt = lib()
    x = _normal((2, 4, 4, 5), 1, 1.0)
    acc = torch.zeros(6, dtype=torch.float64, device=DEV)
    out = sentinel(6)
    dl = sentinel((2, 4, 4, 5))
    gt = torch.ones(1, device=DEV)
    bufs = {"x": x, "acc": acc, "out": out, "dl": dl, "g": gt}
    before = snapshot(bufs)
    lb, st = _C.lib, rt.stream()
    X, A, O, D, G = x.data_ptr(), acc.data_ptr(), out.data_ptr(), dl.data_ptr(), gt.data_ptr()
    calls = [
        ("reduce null logits", lb.pnp_entropy_reduce(None, 32, 5, A, st)),
        ("reduce null acc", lb.pnp_entropy_reduce(X, 32, 5, None, st)),
        ("reduce P 0", lb.pnp_entropy_reduce(X, 0, 5, A, st)),
        ("reduce P -1", lb.pnp_entropy_reduce(X, -1, 5, A, st)),
        ("reduce C 0", lb.pnp_entropy_reduce(X, 32, 0, A, st)),
        ("reduce C 1", lb.pnp_entropy_reduce(X, 32, 1, A, st)),
        ("reduce C 9", lb.pnp_entropy_reduce(X, 32, 9, A, st)),
        ("finalize null acc", lb.pnp_entropy_finalize(None, 32, 5, O, st)),
        ("finalize null out", lb.pnp_entropy_finalize(A, 32, 5, None, st)),
        ("finalize P 0", lb.pnp_entropy_finalize(A, 0, 5, O, st)),
        ("finalize C 1", lb.pnp_entropy_finalize(A, 32, 1, O, st)),
        ("finalize C 9", lb.pnp_entropy_finalize(A, 32, 9, O, st)),
        ("bwd null logits", lb.pnp_entropy_bwd(None, G, D, 32, 5, st)),
        ("bwd null g", lb.pnp_entropy_bwd(X, None, D, 32, 5, st)),
        ("bwd null dlogits", lb.pnp_entropy_bwd(X, G, None, 32, 5, st)),
        ("bwd P 0", lb.pnp_entropy_bwd(X, G, D, 0, 5, st)),
        ("bwd P -7", lb.pnp_entropy_bwd(X, G, D, -7, 5, st)),
        ("bwd C 1", lb.pnp_entropy_bwd(X, G, D, 32, 1, st)),
        ("bwd C 9", lb.pnp_entropy_bwd(X, G, D, 32, 9, st)),
    ]
    for tag, rc in calls:
        assert rc == BAD_ARG, (tag, rc)
    assert_untouched("entropy", "rejected calls", bufs, before)


def test_entropy_loss_autograd_matches_the_oracle():
    """functional.entropy_loss: the loss, p-bar and the gradient autograd hands back, for an upstream gradient of 2.5"""
    lib()
    from pnp_b200 import functional as F
    x = _normal((2, 16, 16, 5), 9, 2.0).requires_grad_(True)
    loss, pbar = F.entropy_loss(x)
    assert not pbar.requires_grad
    (2.5 * loss).backward()
    xn = x.detach().cpu().numpy()
    L, pb, d, _ = E.entropy(xn, 2.5)
    bL, bp, bd = E.bounds(xn, 2.5)
    assert abs(float(loss) - L) <= bL
    assert np.all(np.abs(pbar.cpu().double().numpy() - pb) <= bp)
    assert np.all(np.abs(x.grad.cpu().double().numpy() - d) <= bd)
