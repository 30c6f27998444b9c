"""pnp_bn_accumulate / pnp_bn_population (elementwise.cu) bit for bit against oracle/bn_population_exact.py, at the C-ABI:
C of 1, 3, 16, 512 and 1024, tables of 1 and 60 entries (one launch and past the 64-entry parameter block), count 1 (no
Bessel factor), a NaN channel, a clamped negative variance, k accumulate launches in a row and replayed from a captured
graph; every rejected argument returns PNP_ERR_BAD_ARG and leaves the buffers untouched."""
import numpy as np
import pytest
import torch

from oracle import bn_population_exact as E
from tests.cabi import BAD_ARG, DEV, assert_bits, assert_untouched, lib, snapshot

pytestmark = pytest.mark.gpu


def _f64_equal(tag, got, ref):
    got = got.detach().cpu().contiguous().view(torch.int64)
    ref = torch.from_numpy(np.ascontiguousarray(ref, np.float64)).view(torch.int64)
    bad = (got != ref).nonzero()
    assert bad.numel() == 0, "%s: %d of %d fp64 elements differ, first at %d" % (tag, bad.numel(), got.numel(), int(bad[0]))


class Layer:
    """one entry: per-pass sums, the accumulator and the moving statistics (NaN sentinels: population writes all of them)"""

    def __init__(self, C, rng):
        self.C = C
        self.acc = torch.from_numpy(rng.randn(2 * C) * 10.0).to(DEV)          # a running accumulator need not start at 0
        self.mm = torch.full((C,), float("nan"), device=DEV)
        self.mv = torch.full((C,), float("nan"), device=DEV)

    def pass_sums(self, rng, M):
        """fp64 sums of M values around a channel mean, as a layer's forward would hand them over"""
        mu = rng.randn(self.C) * 2.0
        s1 = mu * M + rng.randn(self.C) * np.sqrt(M)
        s2 = (mu * mu + 1.0) * M + rng.randn(self.C) * np.sqrt(M) * 3.0
        return torch.from_numpy(s1).to(DEV), torch.from_numpy(s2).to(DEV)


def _acc_table(_C, layers, sums):
    t = (_C.BnAccEntry * len(layers))()
    for i, (L, (s1, s2)) in enumerate(zip(layers, sums)):
        t[i] = _C.BnAccEntry(s1.data_ptr(), s2.data_ptr(), L.acc.data_ptr(), L.C)
    return t


def _pop_table(_C, layers, counts):
    t = (_C.BnPopEntry * len(layers))()
    for i, (L, n) in enumerate(zip(layers, counts)):
        t[i] = _C.BnPopEntry(L.acc.data_ptr(), n, L.mm.data_ptr(), L.mv.data_ptr(), L.C)
    return t


CS = [1, 3, 16, 512, 1024]


@pytest.mark.parametrize("n_entries", [1, 60, 130])
@pytest.mark.parametrize("k", [1, 5])
def test_accumulate_then_population_match_the_oracle(n_entries, k):
    _C, rt = lib()
    rng = np.random.RandomState(n_entries * 7 + k)
    layers = [Layer(CS[i % len(CS)] if n_entries > 1 else 1024, rng) for i in range(n_entries)]
    ref = [L.acc.cpu().numpy() for L in layers]
    M = 8 * 16 * 16
    for p in range(k):
        sums = [L.pass_sums(rng, M) for L in layers]
        _C.call("pnp_bn_accumulate", _acc_table(_C, layers, sums), n_entries, rt.stream())
        ref = [E.accumulate(r, s1.cpu().numpy(), s2.cpu().numpy()) for r, (s1, s2) in zip(ref, sums)]
    torch.cuda.synchronize()
    for i, (L, r) in enumerate(zip(layers, ref)):
        _f64_equal("acc entry %d (C %d) after %d passes" % (i, L.C, k), L.acc, r)
    counts = [int(rng.choice([1, 2, k * M, 3 * k * M + 1])) for _ in layers]
    _C.call("pnp_bn_population", _pop_table(_C, layers, counts), n_entries, rt.stream())
    torch.cuda.synchronize()
    for i, (L, r, n) in enumerate(zip(layers, ref, counts)):
        m, v = E.population(r, n)
        assert_bits("moving_mean entry %d (C %d, n %d)" % (i, L.C, n), L.mm.cpu(), torch.from_numpy(m))
        assert_bits("moving_var entry %d (C %d, n %d)" % (i, L.C, n), L.mv.cpu(), torch.from_numpy(v))


def test_population_edge_values():
    """count 1 (no Bessel factor), a NaN channel, an infinite channel, a negative v clamped to 0, v exactly 0"""
    _C, rt = lib()
    rng = np.random.RandomState(0)
    L = Layer(6, rng)
    a1 = np.array([3.0, np.nan, 1.0, 2.0, np.inf, 5.0])
    a2 = np.array([4.0, 1.0, np.nan, 3.0, 1.0, 25.0])                        # channel 0: 4 - 9 < 0; channel 5: v = 0
    for n in (1, 2, 1000):
        acc = np.concatenate([a1, a2]) * n
        L.acc.copy_(torch.from_numpy(acc))
        _C.call("pnp_bn_population", _pop_table(_C, [L], [n]), 1, rt.stream())
        torch.cuda.synchronize()
        m, v = E.population(acc, n)
        assert_bits("mean n=%d" % n, L.mm.cpu(), torch.from_numpy(m))
        assert_bits("var n=%d" % n, L.mv.cpu(), torch.from_numpy(v))
        assert float(L.mv[0]) == 0.0 and np.isnan(float(L.mv[1])) and np.isnan(float(L.mv[2]))


def test_graph_replays_accumulate_k_passes():
    """a captured accumulate launch keeps its table: k replays add the same sums k times, in order"""
    _C, rt = lib()
    rng = np.random.RandomState(4)
    layers = [Layer(c, rng) for c in CS]
    sums = [L.pass_sums(rng, 512) for L in layers]
    table = _acc_table(_C, layers, sums)
    ref = [L.acc.cpu().numpy() for L in layers]
    _C.call("pnp_bn_accumulate", table, len(layers), rt.stream())     # loaded before the capture
    ref = [E.accumulate(r, s1.cpu().numpy(), s2.cpu().numpy()) for r, (s1, s2) in zip(ref, sums)]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _C.call("pnp_bn_accumulate", table, len(layers), rt.stream())
    torch.cuda.synchronize()
    for L, r in zip(layers, ref):
        _f64_equal("acc C %d: capturing runs nothing" % L.C, L.acc, r)
    for k in range(4):
        g.replay()
        ref = [E.accumulate(r, s1.cpu().numpy(), s2.cpu().numpy()) for r, (s1, s2) in zip(ref, sums)]
    torch.cuda.synchronize()
    for L, r in zip(layers, ref):
        _f64_equal("acc C %d after 5 passes" % L.C, L.acc, r)


def test_rejected_arguments():
    _C, rt = lib()
    rng = np.random.RandomState(2)
    L = Layer(16, rng)
    s1, s2 = L.pass_sums(rng, 64)
    bufs = {"acc": L.acc, "mm": L.mm, "mv": L.mv, "s1": s1, "s2": s2}
    before = snapshot(bufs)
    st = rt.stream()
    lb = _C.lib

    def acc(**kw):
        e = dict(sum=s1.data_ptr(), sumsq=s2.data_ptr(), acc=L.acc.data_ptr(), C=16)
        e.update(kw)
        t = (_C.BnAccEntry * 2)(_C.BnAccEntry(s1.data_ptr(), s2.data_ptr(), L.acc.data_ptr(), 16), _C.BnAccEntry(**e))
        return lb.pnp_bn_accumulate(t, 2, st)

    def pop(**kw):
        e = dict(acc=L.acc.data_ptr(), count=64, moving_mean=L.mm.data_ptr(), moving_var=L.mv.data_ptr(), C=16)
        e.update(kw)
        t = (_C.BnPopEntry * 2)(_C.BnPopEntry(L.acc.data_ptr(), 64, L.mm.data_ptr(), L.mv.data_ptr(), 16), _C.BnPopEntry(**e))
        return lb.pnp_bn_population(t, 2, st)

    good_acc = (_C.BnAccEntry * 1)(_C.BnAccEntry(s1.data_ptr(), s2.data_ptr(), L.acc.data_ptr(), 16))
    good_pop = (_C.BnPopEntry * 1)(_C.BnPopEntry(L.acc.data_ptr(), 64, L.mm.data_ptr(), L.mv.data_ptr(), 16))
    calls = [
        ("accumulate null table", lb.pnp_bn_accumulate(None, 1, st)),
        ("accumulate n 0", lb.pnp_bn_accumulate(good_acc, 0, st)),
        ("accumulate n -1", lb.pnp_bn_accumulate(good_acc, -1, st)),
        ("accumulate null sum", acc(sum=None)),
        ("accumulate null sumsq", acc(sumsq=None)),
        ("accumulate null acc", acc(acc=None)),
        ("accumulate C 0", acc(C=0)),
        ("accumulate C -3", acc(C=-3)),
        ("accumulate C 1025", acc(C=1025)),
        ("population null table", lb.pnp_bn_population(None, 1, st)),
        ("population n 0", lb.pnp_bn_population(good_pop, 0, st)),
        ("population null acc", pop(acc=None)),
        ("population null mean", pop(moving_mean=None)),
        ("population null var", pop(moving_var=None)),
        ("population C 0", pop(C=0)),
        ("population C 1025", pop(C=1025)),
        ("population count 0", pop(count=0)),
        ("population count -5", pop(count=-5)),
    ]
    for tag, rc in calls:
        assert rc == BAD_ARG, (tag, rc)
    assert_untouched("bn population", "rejected calls", bufs, before)
