"""The entropy objective without a GPU: oracle/entropy_exact.py against torch fp64 autograd of -(softmax * log_softmax).sum(-1)
.mean() and against central finite differences, each restated mistake changing some output, the a-priori bound's shape, and
adapt_entropy.py's command-line refusals."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import entropy_exact as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _logits(seed, shape, scale):
    return (np.random.RandomState(seed).randn(*shape) * scale).astype(np.float32)


def _torch_ref(x, g=1.0):
    t = torch.from_numpy(x.astype(np.float64)).requires_grad_(True)
    H = -(torch.softmax(t, -1) * torch.log_softmax(t, -1)).sum(-1)
    L = H.mean()
    (g * L).backward()
    return float(L.detach()), torch.softmax(t, -1).reshape(-1, x.shape[-1]).mean(0).detach().numpy(), t.grad.numpy()


@pytest.mark.parametrize("C", [2, 5, 8])
@pytest.mark.parametrize("shape,scale", [((1, 1, 1), 1.0), ((2, 7, 9), 3.0), ((3, 4, 4), 30.0)])
def test_oracle_equals_torch_fp64_autograd(C, shape, scale):
    x = _logits(C + shape[1], shape + (C,), scale)
    L, pbar, d, _ = E.entropy(x, 2.5)
    rL, rp, rd = _torch_ref(x, 2.5)
    assert abs(L - rL) <= 1e-12
    np.testing.assert_allclose(pbar, rp, rtol=0, atol=1e-12)
    np.testing.assert_allclose(d, rd, rtol=0, atol=1e-12)


def test_oracle_gradient_agrees_with_central_differences():
    x = _logits(3, (2, 3, 3, 5), 2.0)
    _, _, d, _ = E.entropy(x)
    x64 = x.astype(np.float64)
    h = 1e-6

    def loss(z):
        m = z.max(-1, keepdims=True)
        t = z - m
        lp = t - np.log(np.exp(t).sum(-1, keepdims=True))
        return -(np.exp(lp) * lp).sum(-1).mean()

    fd = np.empty_like(x64)
    for i in np.ndindex(x64.shape):
        zp, zm = x64.copy(), x64.copy()
        zp[i] += h
        zm[i] -= h
        fd[i] = (loss(zp) - loss(zm)) / (2 * h)
    np.testing.assert_allclose(d, fd, rtol=0, atol=1e-8)


def test_tied_and_saturated_pixels():
    C = 5
    tied = np.full((1, 1, 3, C), 7.0, np.float32)
    L, pbar, d, H = E.entropy(tied)
    assert abs(L - np.log(C)) <= 1e-15 and np.all(np.abs(pbar - 1.0 / C) <= 1e-15) and np.all(np.abs(d) <= 1e-15)
    sat = np.zeros((1, 1, 2, C), np.float32)
    sat[..., 2] = 200.0
    L, _, d, H = E.entropy(sat)
    assert np.all(np.isfinite(d)) and 0.0 <= L <= 1e-80


@pytest.mark.parametrize("flag", ["no_max", "per_batch", "drop_h", "clamp"])
def test_each_restated_mistake_changes_some_output(flag):
    x = _logits(5, (2, 8, 8, 5), 4.0)
    x[0, 0, 0, 1] = 95.0                       # above fp32 exp's overflow at 88.7
    ref = E.entropy(x)
    mut = E.entropy(x, **{flag: True})
    changed = [not np.array_equal(a, b, equal_nan=False) for a, b in zip(ref[:3], mut[:3])]
    assert any(changed), flag


def test_bound_is_a_few_roundings_and_infinite_for_nan():
    a = _logits(1, (1, 4, 4, 5), 1.0)
    bL, bp, bd = E.bounds(a)
    L, pbar, d, _ = E.entropy(a)
    assert 0.0 < bL < 64 * E.U * L and np.all(bp > 0) and np.all(bp < 64 * E.U * pbar)
    assert np.all(bd > 0) and np.all(bd < 1e-3 * np.abs(d).max())
    a[0, 1, 1, 2] = np.nan
    bL, bp, bd = E.bounds(a)
    assert np.isinf(bL) and np.all(np.isinf(bp)) and np.all(np.isinf(bd[0, 1, 1]))


def _cli(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "adapt_entropy.py")] + list(args), cwd=ROOT, capture_output=True,
                          text=True, timeout=600)


@pytest.mark.parametrize("extra,msg", [
    (["--out", "in.npz"], "--out must differ"),
    (["--out", "out.pt"], "--out must name an .npz"),
    (["--steps", "0"], "--steps must be"),
    (["--lr", "0"], "--lr must be positive"),
    (["--lr=-1e-4"], "--lr must be positive"),
    (["--lr", "nan"], "--lr must be positive"),
    (["--batch-size", "0"], "--batch-size must be"),
    (["--recalibrate-batches", "0"], "--recalibrate-batches must be"),
])
def test_cli_refusals(tmp_path, extra, msg):
    base = {"--trainer": "gan", "--checkpoint": str(tmp_path / "in.npz"), "--out": str(tmp_path / "out.npz"),
            "--volumes": str(tmp_path / "pairs.txt")}
    if extra[0] == "--out":
        base["--out"] = str(tmp_path / extra[1])
        extra = []
    args = [a for kv in base.items() for a in kv] + extra
    r = _cli(*args)
    assert r.returncode == 2, r.stderr
    assert msg in r.stderr, r.stderr
    assert not os.path.exists(tmp_path / "out.npz")


def test_cli_needs_one_source(tmp_path):
    r = _cli("--trainer", "segmenter", "--checkpoint", str(tmp_path / "a.npz"), "--out", str(tmp_path / "b.npz"))
    assert r.returncode == 2 and "--volumes" in r.stderr


def test_log_layout(tmp_path):
    import pnp_b200  # noqa: F401  (the package alias; tent imports no CUDA at module level beyond the library handle)
    from pnp_b200 import tent
    assert tent.log_path("/a/b/out.npz") == "/a/b/out_entropy.csv"
    h = np.array([[1.5, 0.2, 0.8], [1.25, 0.3, 0.7]], np.float32)
    p = tmp_path / "x_entropy.csv"
    tent.write_log(str(p), h)
    rows = p.read_text().splitlines()
    assert rows[0] == "step,entropy,pbar_0,pbar_1"
    assert len(rows) == 3 and rows[2].startswith("1,1.25,")
