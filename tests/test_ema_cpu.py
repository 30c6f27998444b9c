"""The reference of the weights' moving average (oracle/ema_exact.py) and the host side of the opt-in EMA, without a GPU:
* the fp32 decay schedule is TF's formula for n = 0, 1, 9, 10^4 and 2^24 +- 1 at decays 0.5, 0.999 and 0.9999, against a
  restatement that rounds an fp64 evaluation of each operation to fp32 (exact for one addition or division of fp32 values);
* each mutation of the oracle (the d*s + (1-d)*x form, a contracted FMA, the decay in fp64, n off by one) changes some output
  on the designed inputs below, so the GPU tests that hold the kernels to the oracle would see it;
* the command-line rules of --ema-decay;
* lib.save_checkpoint's files and key sets, with a stub trainer."""
import os

import numpy as np
import pytest

from oracle import ema_exact as E

f32 = np.float32
NS = [0, 1, 9, 10 ** 4, (1 << 24) - 1, 1 << 24, (1 << 24) + 1]
DECAYS = [0.5, 0.999, 0.9999]


def _rn(v):
    """fp64 -> nearest fp32"""
    return f32(np.float64(v))


def _schedule_ref(n, decay):
    nf = _rn(float(n))                       # float(n) is exact below 2^53
    q = _rn(np.float64(_rn(1.0 + np.float64(nf))) / np.float64(_rn(10.0 + np.float64(nf))))
    d = min(f32(decay), q)
    return _rn(1.0 - np.float64(d))


@pytest.mark.parametrize("decay", DECAYS)
def test_decay_schedule(decay):
    for n in NS:
        c, n1 = E.advance(n, decay)
        assert n1 == n + 1 and c.dtype == np.float32
        assert c == _schedule_ref(n, decay), (n, decay, c)
    # the hand-checked points: d = 1/10 at n = 0, d = decay once the warm-up ratio passes it; 2^24 + 1 rounds to 2^24
    assert E.advance(0, decay)[0] == f32(1.0) - f32(0.1)
    assert E.advance(1 << 24, decay)[0] == f32(1.0) - f32(decay)
    assert E.advance((1 << 24) + 1, decay)[0] == E.advance(1 << 24, decay)[0]
    assert E.advance(9, 0.5)[0] == f32(0.5)


def _designed():
    """shadows and live values over 16 binades, the live values near the shadows (as after one optimizer step) and far"""
    rng = np.random.RandomState(7)
    s = (rng.randn(8192) * np.exp2(rng.randint(-8, 8, 8192))).astype(np.float32)
    x = np.where(np.arange(8192) % 2 == 0, s * (1 + 1e-3 * rng.randn(8192)), rng.randn(8192)).astype(np.float32)
    lives = [x, (x * f32(1.001)).astype(np.float32), (x - f32(0.25)).astype(np.float32)]
    return s, lives


@pytest.mark.parametrize("mutation", [{"form": "blend"}, {"fma": True}, {"decay_fp64": True}, {"n_offset": 1}, {"n_offset": -1}],
                         ids=["blend_form", "fma", "decay_fp64", "n_plus_1", "n_minus_1"])
def test_mutations_change_the_output(mutation):
    s, lives = _designed()
    changed = False
    for decay in DECAYS:
        for n0 in (1, 9, 11, 17, 100):
            ref, _ = E.steps(s, lives, n0, decay)
            got, _ = E.steps(s, lives, n0, decay, **mutation)
            changed |= not np.array_equal(ref.view(np.int32), got.view(np.int32))
    assert changed, mutation


def test_update_and_swap_basics():
    s, lives = _designed()
    out, n = E.steps(s, lives, 0, 0.999)
    assert n == 3 and out.dtype == np.float32
    # c = 1 - d is exact, so with x == s the shadow stays put bit for bit
    assert np.array_equal(E.update(s, s, E.advance(5, 0.9)[0]), s)
    a, b = E.swap(s, lives[0])
    assert np.array_equal(a, lives[0]) and np.array_equal(b, s)
    a2, b2 = E.swap(a, b)
    assert np.array_equal(a2.view(np.int32), s.view(np.int32)) and np.array_equal(b2.view(np.int32), lives[0].view(np.int32))


def test_command_line_rules():
    import pnp_b200  # noqa: F401
    from pnp_b200 import train_segmenter, train_gan
    for bad in ("0", "1", "-0.5", "1.5", "nan"):
        with pytest.raises(SystemExit):
            train_segmenter.main(["--synthetic", "--ema-decay", bad])
        with pytest.raises(SystemExit):
            train_gan.main("train-gan", ["--phase", "train-gan", "--synthetic", "--ema-decay", bad])
    with pytest.raises(SystemExit):
        train_gan.main("pre-train", ["--phase", "pre-train", "--synthetic", "--ema-decay", "0.999"])


class _DP:
    def save_checkpoint(self, fn):
        fn()


class _StubTrainer:
    def __init__(self, state, ema):
        self.state, self.ema, self.global_step, self.dp = state, ema, 7, _DP()

    def checkpoint_state(self):
        return dict(self.state)


def _stub_graph():
    import torch
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt
    rt.reset_default_graph()
    for name in ("adapt_1/Variable", "adapt_1/adapt_1_1/moving_mean", "cls_scope/cls_1/Variable"):
        rt.get_variable(name, lambda: torch.zeros(3))
    return rt


@pytest.mark.parametrize("with_ema", [False, True])
def test_save_checkpoint_files_and_keys(tmp_path, with_ema):
    from pnp_b200 import ema as ema_mod
    from pnp_b200.lib import save_checkpoint
    rt = _stub_graph()
    live = {n: np.full(3, i, np.float32) for i, n in enumerate(rt.graph.order)}
    st = dict(live)
    st.update({"adapt_1/Variable/RMSProp": np.ones(3, np.float32), "pnp/learning_rate": np.float32(3e-4),
               "pnp/global_step": np.int64(7)})
    if with_ema:
        shadows = {n: np.full(3, 10 + i, np.float32) for i, n in enumerate(rt.graph.order[:2])}
        st.update({n + ema_mod.SUFFIX: v for n, v in shadows.items()})
        st.update({ema_mod.NUM_UPDATES_KEY: np.int64(5), ema_mod.DECAY_KEY: np.float32(0.999)})
    out = str(tmp_path)
    save_checkpoint(_StubTrainer(st, object() if with_ema else None), os.path.join(out, "model.cpkt"), out)
    want = {"model.cpkt-7.npz", "latest.npz"} | ({"model.cpkt-7_ema.npz", "latest_ema.npz"} if with_ema else set())
    assert set(os.listdir(out)) == want
    for f in ("model.cpkt-7.npz", "latest.npz"):
        d = np.load(os.path.join(out, f))
        assert set(d.files) == set(st)
    if with_ema:
        for f in ("model.cpkt-7_ema.npz", "latest_ema.npz"):
            d = np.load(os.path.join(out, f))
            assert set(d.files) == set(rt.graph.order) | {"pnp/global_step"}
            for n in rt.graph.order:
                assert np.array_equal(d[n], shadows.get(n, live[n])), n
            assert int(d["pnp/global_step"]) == 7


def test_decay_is_checked_on_the_host():
    from pnp_b200.ema import check_decay
    for bad in (0.0, 1.0, -1.0, float("nan")):
        with pytest.raises(ValueError):
            check_decay(bad)
    assert check_decay(0.999) == 0.999
