"""pnp_ema_advance / pnp_ema_update / pnp_ema_swap (elementwise.cu) bit for bit against oracle/ema_exact.py, at the C-ABI:
arena-shaped buffers with padding, tables of tensors of length 1, 1023, 1024 and 1025 and of many segments, n = 0 and large n,
a single CTA and many CTAs, k replays of a captured graph of both launches; two swaps are the identity; every rejected argument
returns PNP_ERR_BAD_ARG and leaves the buffers untouched."""
import numpy as np
import pytest
import torch

from oracle import ema_exact as E
from tests.cabi import BAD_ARG, DEV, assert_bits, assert_untouched, lib, ptr, snapshot

pytestmark = pytest.mark.gpu
CH = 1024


class Case:
    """a live arena of `arena_vars` variables (each padded to 1024 floats, padding zero) and `extra` separate tensors, their
    shadow and chunk table"""

    def __init__(self, arena_vars, extra, seed):
        g = torch.Generator().manual_seed(seed)
        self.arena_n = sum(-(-n // CH) * CH for n in arena_vars)
        theta = torch.zeros(self.arena_n)
        off = 0
        for n in arena_vars:
            theta[off:off + n] = torch.randn(n, generator=g) * 2.0 ** torch.randint(-6, 6, (n,), generator=g)
            off += -(-n // CH) * CH
        self.theta = theta.to(DEV)
        self.extra = [(torch.randn(n, generator=g) * 0.5 + 1.0).to(DEV) for n in extra]
        entries = []
        for t in self.extra:
            for j in range(0, t.numel(), CH):
                entries.append((t.data_ptr() + 4 * j, min(CH, t.numel() - j)))
        self.table_n = len(entries)
        self.table = torch.tensor(entries, dtype=torch.int64, device=DEV).reshape(-1, 2) if entries else None
        self.total = self.arena_n + CH * self.table_n
        # the shadow starts away from the live values; the extra segments' padding holds values nobody may touch
        self.shadow = (torch.randn(self.total, generator=g)).to(DEV)
        self.n = torch.zeros(1, dtype=torch.int64, device=DEV)
        self.c = torch.zeros(1, dtype=torch.float32, device=DEV)

    def live_flat(self):
        """the live values in shadow layout (extra padding: the shadow's own, which the kernels never change)"""
        out = self.shadow.clone()
        out[:self.arena_n] = self.theta
        k = self.arena_n
        for t in self.extra:
            nch = -(-t.numel() // CH)
            out[k:k + t.numel()] = t
            k += nch * CH
        return out

    def covered(self):
        """mask of the shadow floats that mirror a live float (arena padding included)"""
        m = torch.zeros(self.total, dtype=torch.bool)
        m[:self.arena_n] = True
        k = self.arena_n
        for t in self.extra:
            m[k:k + t.numel()] = True
            k += -(-t.numel() // CH) * CH
        return m

    def advance(self, _C, rt, decay):
        _C.call("pnp_ema_advance", ptr(self.n), decay, ptr(self.c), rt.stream())

    def update(self, _C, rt):
        _C.call("pnp_ema_update", ptr(self.shadow), ptr(self.theta), self.arena_n, ptr(self.table), self.table_n, ptr(self.c), rt.stream())

    def swap(self, _C, rt):
        _C.call("pnp_ema_swap", ptr(self.shadow), ptr(self.theta), self.arena_n, ptr(self.table), self.table_n, rt.stream())

    def perturb(self, step):
        """what an optimizer step does to the live values (deterministic, on the device)"""
        with torch.no_grad():
            self.theta.mul_(1.0 + 1e-3 * (step + 1))
            for t in self.extra:
                t.add_(0.01 * (step + 1))


def oracle_step(case, s, n, decay, live):
    cov = case.covered().numpy()
    c, n1 = E.advance(n, decay)
    out = s.copy()
    out[cov] = E.update(s[cov], live[cov], c)
    return out, n1, c


CASES = [
    ("one_cta", [1000], [], 0, 0.999),
    ("padding", [1, 1023, 1024, 1025], [], 0, 0.9999),
    ("table_lengths", [1025], [1, 1023, 1024, 1025], 0, 0.5),
    ("many_segments", [3 * 3 * 64 * 64, 7], [int(x) for x in np.random.RandomState(3).randint(1, 3000, 150)], 0, 0.999),
    ("large_n", [5000], [64, 2049], (1 << 24) + 1, 0.9999),
    ("many_ctas", [1 << 20, 1 << 20], [32] * 40, 12345, 0.999),
]


@pytest.mark.parametrize("arena_vars,extra,n0,decay", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_advance_update_match_the_oracle(arena_vars, extra, n0, decay):
    _C, rt = lib()
    case = Case(arena_vars, extra, seed=len(extra) + n0 % 97)
    case.n.fill_(n0)
    s, n = case.shadow.cpu().numpy(), n0
    for k in range(4):
        live = case.live_flat().cpu().numpy()
        case.advance(_C, rt, decay)
        case.update(_C, rt)
        s, n, c = oracle_step(case, s, n, decay, live)
        torch.cuda.synchronize()
        assert int(case.n.item()) == n
        assert_bits("c step %d" % k, case.c.cpu(), torch.tensor([c]))
        assert_bits("shadow step %d" % k, case.shadow.cpu(), torch.from_numpy(s))
        case.perturb(k)


def test_graph_replays_advance_n_and_match_k_oracle_steps():
    _C, rt = lib()
    case = Case([1025, 4096], [1, 1025, 3000], seed=11)
    decay = 0.999
    warm = Case([1024], [3], seed=12)              # both kernels loaded before the capture
    warm.advance(_C, rt, decay)
    warm.update(_C, rt)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        case.advance(_C, rt, decay)
        case.update(_C, rt)
    torch.cuda.synchronize()
    assert int(case.n.item()) == 0                 # capturing runs nothing
    sh, n = case.shadow.cpu().numpy(), 0
    for k in range(5):
        live = case.live_flat().cpu().numpy()
        g.replay()
        sh, n, _ = oracle_step(case, sh, n, decay, live)
        torch.cuda.synchronize()
        assert int(case.n.item()) == n == k + 1
        assert_bits("replay %d" % k, case.shadow.cpu(), torch.from_numpy(sh))
        case.perturb(k)


def test_swap_exchanges_and_twice_is_identity():
    _C, rt = lib()
    case = Case([1, 1023, 1025], [1, 1023, 1024, 1025], seed=5)
    s0, live0 = case.shadow.clone(), case.live_flat()
    extra0 = [t.clone() for t in case.extra]
    theta0 = case.theta.clone()
    case.swap(_C, rt)
    torch.cuda.synchronize()
    cov = case.covered().to(DEV)
    assert_bits("shadow after swap", case.shadow[cov], live0[cov])
    assert_bits("padding after swap", case.shadow[~cov], s0[~cov])
    assert_bits("arena after swap", case.theta, s0[:case.arena_n])
    case.swap(_C, rt)
    torch.cuda.synchronize()
    assert_bits("shadow twice", case.shadow, s0)
    assert_bits("arena twice", case.theta, theta0)
    for t, t0 in zip(case.extra, extra0):
        assert_bits("extra twice", t, t0)


def test_rejected_arguments():
    _C, rt = lib()
    case = Case([1024], [5], seed=2)
    bufs = {"shadow": case.shadow, "theta": case.theta, "extra": case.extra[0], "n": case.n, "c": case.c}
    before = snapshot(bufs)
    st = rt.stream()
    L = _C.lib
    sh, th, tb, cc, nn = ptr(case.shadow), ptr(case.theta), ptr(case.table), ptr(case.c), ptr(case.n)
    calls = [
        ("advance null n", L.pnp_ema_advance(None, 0.9, cc, st)),
        ("advance null c", L.pnp_ema_advance(nn, 0.9, None, st)),
    ] + [("advance decay %r" % d, L.pnp_ema_advance(nn, d, cc, st)) for d in (0.0, 1.0, -0.5, 1.5, float("nan"))] + [
        ("update null shadow", L.pnp_ema_update(None, th, 1024, tb, 1, cc, st)),
        ("update null arena", L.pnp_ema_update(sh, None, 1024, tb, 1, cc, st)),
        ("update null c", L.pnp_ema_update(sh, th, 1024, tb, 1, None, st)),
        ("update null table", L.pnp_ema_update(sh, th, 1024, None, 1, cc, st)),
        ("update arena_n 0", L.pnp_ema_update(sh, th, 0, tb, 1, cc, st)),
        ("update arena_n -1024", L.pnp_ema_update(sh, th, -1024, tb, 1, cc, st)),
        ("update arena_n 1000", L.pnp_ema_update(sh, th, 1000, tb, 1, cc, st)),
        ("update table_n -1", L.pnp_ema_update(sh, th, 1024, tb, -1, cc, st)),
        ("update too many chunks", L.pnp_ema_update(sh, th, 1024 << 31, tb, 1, cc, st)),
        ("swap null shadow", L.pnp_ema_swap(None, th, 1024, tb, 1, st)),
        ("swap null arena", L.pnp_ema_swap(sh, None, 1024, tb, 1, st)),
        ("swap null table", L.pnp_ema_swap(sh, th, 1024, None, 1, st)),
        ("swap arena_n 0", L.pnp_ema_swap(sh, th, 0, tb, 1, st)),
        ("swap arena_n 1536", L.pnp_ema_swap(sh, th, 1536, tb, 1, st)),
        ("swap table_n -2", L.pnp_ema_swap(sh, th, 1024, tb, -2, st)),
    ]
    for tag, rc in calls:
        assert rc == BAD_ARG, (tag, rc)
    assert_untouched("ema", "rejected calls", bufs, before)
    # an empty table is allowed (no statistics to average)
    assert L.pnp_ema_update(sh, th, 1024, None, 0, cc, st) == 0
    assert L.pnp_ema_swap(sh, th, 1024, None, 0, st) == 0
    torch.cuda.synchronize()
