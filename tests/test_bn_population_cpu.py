"""The batch-norm population statistics without a GPU: oracle/bn_population_exact.py against an independent two-pass fp64
pooled mean and variance, each restated mistake changing some output, and recalibrate_bn.py's command-line rules and output
key set."""
import numpy as np
import pytest

from oracle import bn_population_exact as E

EPS64 = np.finfo(np.float64).eps


def _passes(seed, N, M, C, mean, std, drift=0.0):
    """N passes of M values per channel; the pass means drift apart by `drift` standard deviations per pass"""
    rng = np.random.RandomState(seed)
    centre = mean * (1.0 + rng.rand(C))
    vals = [(centre + std * (drift * b + rng.randn(M, C))).astype(np.float32) for b in range(N)]
    return vals, [E.batch_sums(z) for z in vals]


@pytest.mark.parametrize("N,M,C", [(1, 2, 3), (7, 8 * 64, 16), (40, 8 * 32 * 32, 8)])
def test_restatement_equals_the_two_pass_reference(N, M, C):
    """Well-conditioned values (|mean| <= 2 std).  The one-pass moments differ from the two-pass ones only by rounding:
    A1 and A2 carry at most (N + log2 M) relative roundings of the sums of |z| and z^2, and v = A2/n - m^2 inherits the
    error of both terms, so |v1 - v2| <= 4 (N + log2 M + 4) eps (A2 / n) and |m1 - m2| <= 4 (N + log2 M + 4) eps (A1abs / n).
    The fp32 outputs are then within one fp32 rounding of the reference's, plus that bound."""
    vals, passes = _passes(3 + N, N, M, C, mean=1.0, std=0.5, drift=0.3)
    acc = np.zeros(2 * C)
    for s1, s2, _ in passes:
        acc = E.accumulate(acc, s1, s2)
    n = N * M
    m1, v1 = E.moments(acc, n)
    m2, v2 = E.two_pass(vals)
    v2_biased = v2 * ((n - 1) / n) if n > 1 else v2
    k = 4 * (N + np.log2(M) + 4) * EPS64
    a1abs = sum(np.abs(z.astype(np.float64)).sum(axis=0) for z in vals)
    assert np.all(np.abs(m1 - m2) <= k * a1abs / n)
    assert np.all(np.abs(v1 - v2_biased) <= k * acc[C:] / n)
    mean, var = E.recalibrate(passes)
    f32 = np.finfo(np.float32).eps
    assert np.all(np.abs(mean - m2) <= f32 * np.abs(m2) + k * a1abs / n)
    assert np.all(np.abs(var - v2) <= f32 * v2 + 2 * k * acc[C:] / n)


def test_the_variance_is_pooled_not_the_mean_of_batch_variances():
    """pooled variance = mean within-pass variance + variance of the pass means"""
    vals, passes = _passes(1, 6, 256, 4, mean=0.0, std=1.0, drift=1.0)
    _, var = E.recalibrate(passes, biased=True)
    within = np.mean([z.astype(np.float64).var(axis=0) for z in vals], axis=0)
    between = np.var([z.astype(np.float64).mean(axis=0) for z in vals], axis=0)
    np.testing.assert_allclose(var, within + between, rtol=1e-5)


def test_count_one_has_no_bessel_factor_and_negative_v_is_clamped():
    mean, var = E.population(np.array([3.0, 0.0, 4.0, -1.0]), 1)       # m = (3, 0), v = (4 - 9, -1) -> clamped
    assert mean.tolist() == [3.0, 0.0] and var.tolist() == [0.0, 0.0]
    mean, var = E.population(np.array([np.nan, 2.0, 1.0, 8.0]), 2)
    assert np.isnan(mean[0]) and np.isnan(var[0]) and var[1] == np.float32((4.0 - 1.0) * 2.0)


MUTATIONS = ["average_variances", "biased", "fma", "fp32", "reverse"]


@pytest.mark.parametrize("flag", MUTATIONS)
def test_each_mutation_changes_some_output(flag):
    """ill-conditioned on purpose (mean 1e4 standard deviations away, drifting pass means): A2 / n - m^2 cancels, so a
    different rounding anywhere upstream reaches the fp32 variance"""
    _, passes = _passes(11, 24, 64, 512, mean=3.0e4, std=1.0, drift=0.5)
    ref = E.recalibrate(passes)
    got = E.recalibrate(passes, **{flag: True})
    changed = sum(int(np.sum(a.view(np.int32) != b.view(np.int32))) for a, b in zip(ref, got))
    assert changed > 0, flag


# ---------------------------------------------------------------------------------------------------------------------------
# recalibrate_bn.py
# ---------------------------------------------------------------------------------------------------------------------------
def _parse(argv):
    from pnp_b200 import bnstats
    ap = bnstats.build_parser()
    a = ap.parse_args(argv)
    bnstats.check_args(a, ap.error)
    return a


@pytest.fixture
def cli():
    pytest.importorskip("torch")
    try:
        import pnp_b200  # noqa: F401
    except ImportError as e:          # the library is built by build(); without it there is nothing to import
        pytest.skip(str(e))
    return _parse


def test_cli_defaults(cli):
    a = cli(["--trainer", "gan", "--checkpoint", "a.npz", "--out", "b.npz", "--volumes", "pairs"])
    assert (a.batches, a.batch_size, a.scope, a.records) == (200, 8, None, None)


@pytest.mark.parametrize("argv", [
    ["--trainer", "gan", "--checkpoint", "a.npz", "--out", "a.npz", "--volumes", "p"],                  # OUT == IN
    ["--trainer", "gan", "--checkpoint", "d/../a.npz", "--out", "a.npz", "--volumes", "p"],             # OUT == IN, spelled apart
    ["--trainer", "segmenter", "--checkpoint", "a.npz", "--out", "b.npz", "--volumes", "p", "--scope", "dam"],
    ["--trainer", "gan", "--checkpoint", "a.npz", "--out", "b.npz"],                                    # no source
    ["--trainer", "gan", "--checkpoint", "a.npz", "--out", "b.npz", "--volumes", "p", "--records", "r"],
    ["--trainer", "gan", "--checkpoint", "a.npz", "--out", "b.npz", "--volumes", "p", "--batches", "0"],
    ["--trainer", "gan", "--checkpoint", "a.npz", "--out", "b.npz", "--volumes", "p", "--scope", "mr"],
    ["--trainer", "gan", "--checkpoint", "a.npz", "--out", "b", "--volumes", "p"],                      # not an .npz
])
def test_cli_refusals(cli, argv):
    with pytest.raises(SystemExit):
        cli(argv)


def test_cli_accepts_scope_all_and_records(cli):
    a = cli(["--trainer", "gan", "--checkpoint", "latest_ema.npz", "--out", "o.npz", "--records", "ct_train_list",
             "--scope", "all", "--batches", "3", "--batch-size", "2", "--seed", "9"])
    assert (a.scope, a.records, a.batches, a.batch_size, a.seed) == ("all", "ct_train_list", 3, 2, 9)


def test_output_key_set(cli):
    """every graph variable and pnp/global_step of the input; no optimizer slot, no EMA key"""
    from pnp_b200 import bnstats, runtime as rt

    class Net:
        last_restored = {"pnp/global_step": np.int64(17), "a/RMSProp": np.zeros(1), "a/ExponentialMovingAverage": np.zeros(1)}

    class Trainer:
        net = Net()

    saved = rt.state_dict
    rt.state_dict = lambda: {"a": np.zeros(1, np.float32), "s/moving_mean": np.ones(2, np.float32)}
    try:
        st = bnstats.recalibrated_checkpoint(Trainer())
    finally:
        rt.state_dict = saved
    assert sorted(st) == ["a", "pnp/global_step", "s/moving_mean"]
    assert int(st["pnp/global_step"]) == 17
