"""The reference of the augmentation kernels (oracle/augment_exact.py) and the host side of the opt-in elastic and intensity
augmentations (preprocess.py, data.VolumeSource, prepare_data and the trainers' flags), without a GPU:
* the fp32 restatement of the smoothed field equals scipy's gaussian_filter1d in fp64 on the same uniforms within an a-priori
  bound, and its taps are scipy's;
* the uniforms are the words of the independent Philox4x32-10 of oracle/philox.py, one by one;
* the field statistics behind the chosen amplitudes (DESIGN 6.1), and the clamps;
* every worst-case sample, deformed by the largest displacement, stays inside the sub-volume built with ELASTIC_REACH_PX;
* with both flags off a VolumeSource consumes its RandomState exactly as before, and with intensity on it draws (a, b) right
  after each sample's (j, T);
* the command-line flags are rejected where they do not apply."""
import math

import numpy as np
import pytest
import scipy.ndimage as nd

from oracle import augment_exact as A
from oracle import philox
from tests import mmwhs_phantom as ph


def _pp():
    import pnp_b200  # noqa: F401
    from pnp_b200 import preprocess
    return preprocess


@pytest.mark.parametrize("sigma", [0.1, 0.7, 2.0, 10.0, 32.0])
def test_taps_are_scipys(sigma):
    t = A.gaussian_taps(sigma)
    r = int(4.0 * sigma + 0.5)
    assert len(t) == 2 * r + 1 and t.dtype == np.float32
    # scipy's own filter of a unit impulse is its fp64 kernel
    imp = np.zeros(4 * r + 3)
    imp[2 * r + 1] = 1.0
    ref = nd.gaussian_filter1d(imp, sigma, mode="constant")[r + 1:3 * r + 2]
    assert np.array_equal(t, ref.astype(np.float32))
    assert np.array_equal(_pp().gaussian_taps(sigma), t)


# (B, K, H, W, sigma): R = 0, R >= W / 2, odd sizes, the production sigmas
FIELD_CASES = [(2, 1, 7, 9, 0.1), (1, 2, 13, 6, 2.0), (2, 2, 40, 37, 10.0), (1, 1, 64, 300, 32.0), (3, 2, 19, 260, 3.0)]


@pytest.mark.parametrize("case", FIELD_CASES, ids=lambda c: "x".join(map(str, c)))
def test_restated_field_equals_scipy_within_the_bound(case):
    B, K, H, W, sigma = case
    taps = A.gaussian_taps(sigma)
    u = A.uniforms(77, 0xE1A5 << 32 | 3, B, K, H, W)
    got = A.smooth(u, taps)
    ref = nd.gaussian_filter1d(nd.gaussian_filter1d(u.astype(np.float64), sigma, axis=-1, mode="constant"), sigma, axis=-2,
                               mode="constant")
    bound = A.smooth_error_bound(taps)
    err = float(np.abs(got.astype(np.float64) - ref).max())
    print("%s: max error %.3e, bound %.3e" % (case, err, bound))
    assert err <= bound
    # amp, lo and hi are one rounding and a clamp
    f = A.noise_field(77, 0xE1A5 << 32 | 3, B, K, H, W, taps, 3.0, -0.01, 0.02)
    assert np.array_equal(f, np.fmin(np.fmax(np.float32(3.0) * got, np.float32(-0.01)), np.float32(0.02)))


def test_uniforms_are_the_philox_words():
    B, K, H, W = 2, 2, 5, 7
    seed, stream = 0x1234_5678_9ABC_DEF0, (0xB1A5 << 32) | 41
    u = A.uniforms(seed, stream, B, K, H, W).reshape(-1)
    n = u.size
    for e in range(n):
        ctr = [(e >> 2) & 0xFFFFFFFF, e >> 34, stream & 0xFFFFFFFF, stream >> 32]
        w = int(philox.philox4x32_10(np.array(ctr), np.array([seed & 0xFFFFFFFF, seed >> 32]))[e & 3])
        assert u[e] == np.float32((w >> 8) * 2.0 ** -23 - 1.0), e         # exact: a 24-bit integer times 2^-23, minus 1
    assert u.min() >= -1.0 and u.max() < 1.0
    # exactness: every value maps back to its 24-bit integer
    k = (u.astype(np.float64) + 1.0) * 2.0 ** 23
    assert np.array_equal(k, np.floor(k))


def test_field_stream_tags():
    pp = _pp()
    assert pp.field_stream(pp.ELASTIC_STREAM_TAG, 5) == 0xE1A5_0000_0005
    assert pp.field_stream(pp.BIAS_STREAM_TAG, 0) == 0xB1A5_0000_0000
    assert pp.ELASTIC_STREAM_TAG != pp.BIAS_STREAM_TAG
    with pytest.raises(ValueError):
        pp.field_stream(pp.BIAS_STREAM_TAG, 1 << 32)


def test_field_statistics_and_clamps():
    """RMS and largest |s| of the smoothed uniforms over 16 planes of 256 x 256 at the two sigmas (the figures DESIGN 6.1 quotes),
    and the clamped fields"""
    pp = _pp()
    te, tb = A.gaussian_taps(pp.ELASTIC_SIGMA), A.gaussian_taps(pp.BIAS_SIGMA)
    assert len(tb) - 1 <= 2 * A.NF_MAX_R
    se = A.smooth(A.uniforms(1234, pp.field_stream(pp.ELASTIC_STREAM_TAG, 0), 8, 2, 256, 256), te)
    sb = A.smooth(A.uniforms(1234, pp.field_stream(pp.BIAS_STREAM_TAG, 0), 16, 1, 256, 256), tb)
    rms_e, max_e = float(np.sqrt((se.astype(np.float64) ** 2).mean())), float(np.abs(se).max())
    rms_b = float(np.sqrt((sb.astype(np.float64) ** 2).mean()))
    print("elastic s: rms %.4f max %.4f; bias s: rms %.4f" % (rms_e, max_e, rms_b))
    assert 0.014 < rms_e < 0.018 and max_e < 0.08
    assert 0.08 < pp.BIAS_BETA * rms_b < 0.12
    assert pp.ELASTIC_ALPHA * max_e < pp.ELASTIC_MAX_PX            # the clamp practically never binds
    # the clamps: a large amplitude saturates at both bounds and never beyond
    d = A.noise_field(9, 1, 2, 2, 32, 32, te, 1e4, -pp.ELASTIC_MAX_PX, pp.ELASTIC_MAX_PX)
    assert d.max() == pp.ELASTIC_MAX_PX and d.min() == -pp.ELASTIC_MAX_PX
    g = A.noise_field(9, 2, 2, 1, 64, 64, te, 1e4, -pp.BIAS_MAX, pp.BIAS_MAX)
    gain = np.float32(1) + g
    assert gain.min() == 0.5 and gain.max() == 1.5
    assert pp.ELASTIC_REACH_PX == pp.REACH_PX + pp.SCALE_RANGE[1] * math.sqrt(2.0) * pp.ELASTIC_MAX_PX


@pytest.fixture(scope="module")
def subjects(tmp_path_factory):
    pp = _pp()
    d = str(tmp_path_factory.mktemp("aug_cpu"))
    pairs = ph.write_pairs(d, "ct", [31, 32], spacing=(0.8, 1.3, 1.1)) + ph.write_pairs(d, "mr", [33], shape=(40, 52, 30),
                                                                                            spacing=(1.2, 0.7, 1.6))
    return pairs, [pp.Subject(im, lb, reach_px=pp.ELASTIC_REACH_PX) for im, lb in pairs]


def test_worst_case_deformed_samples_stay_inside_the_enlarged_sub_volume(subjects):
    """every corner and edge-midpoint pixel, displaced by (+-D_max, +-D_max), under the extreme rotations, scales and shifts,
    at the first and last slice: every coordinate lies inside [0, n - 1] of the sub-volume, in fp64 and in the kernel's fp32"""
    pp = _pp()
    _, subs = subjects
    S, D = pp.SIZE, pp.ELASTIC_MAX_PX
    pix = np.array([(r, c) for r in (0, S / 2, S - 1) for c in (0, S / 2, S - 1)], np.float64)
    disp = np.array([(a, b) for a in (-D, 0, D) for b in (-D, 0, D)], np.float64)
    worst = []
    for th in np.linspace(-pp.ROTATION_DEG, pp.ROTATION_DEG, 7):
        for s0 in pp.SCALE_RANGE:
            for s1 in pp.SCALE_RANGE:
                for t0 in (-pp.SHIFT_PX, pp.SHIFT_PX):
                    for t1 in (-pp.SHIFT_PX, pp.SHIFT_PX):
                        a = np.deg2rad(th)
                        A2 = np.array([[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]]) @ np.diag([s0, s1])
                        T = np.eye(3)
                        T[:2, :2] = A2
                        T[:2, 2] = pp.CENTRE + np.array([t0, t1]) - A2 @ np.array([pp.CENTRE, pp.CENTRE])
                        worst.append(T)
    for s in subs:
        n = np.array(s.vol.shape)
        for j in (s.j_lo, s.j_hi):
            for T in worst:
                m64 = s.base(j) @ T
                m32 = s.matrices((j,), T)[0]
                for p in pix:
                    for d in disp:
                        q = p + d
                        u = m64 @ np.array([q[0], q[1], 1.0])
                        assert np.all(u >= 0) and np.all(u <= n - 1), (s.name, j, u, n)
                        qf = np.float32(q[0]), np.float32(q[1])
                        uf = [(m32[i, 0] * qf[0] + m32[i, 1] * qf[1]) + m32[i, 2] for i in range(3)]
                        assert all(0 <= uf[i] <= n[i] - 1 for i in range(3)), (s.name, j, uf, n)
    # the default reach does not contain them: the enlargement is needed
    im, lb = subjects[0][0]
    plain = pp.Subject(im, lb)
    assert plain.vol.shape[1] < subs[0].vol.shape[1] and plain.vol.shape[2] < subs[0].vol.shape[2]


def _bare_source(subs, B, seed, augment=True, intensity=False):
    """a VolumeSource's host drawing state without the device buffers"""
    import pnp_b200  # noqa: F401
    from pnp_b200.data import VolumeSource
    v = VolumeSource.__new__(VolumeSource)
    v.B, v.augment, v.elastic, v.intensity = B, augment, False, intensity
    v.subjects, v.offsets = subs, [0, 100, 200][:len(subs)]
    v.rng = np.random.RandomState(seed)
    return v


def test_flags_off_consume_the_generator_as_before(subjects):
    _, subs = subjects
    for augment in (True, False):
        v = _bare_source(subs, 5, 99, augment)
        rng = np.random.RandomState(99)
        for _ in range(3):
            want = []
            for _ in range(5):                        # the draw order of VolumeSource.draw_matrices before the flags existed
                s = int(rng.randint(len(subs)))
                j, T = subs[s].draw(rng, augment)
                want.append(subs[s].matrices((j - 1, j, j + 1), T, v.offsets[s]))
            mats, ab = v.draw_samples()
            assert ab is None and np.array_equal(mats, np.stack(want))
        assert rng.randint(1 << 30) == v.rng.randint(1 << 30)
        v2 = _bare_source(subs, 5, 99, augment)
        assert np.array_equal(v2.draw_matrices(), _bare_source(subs, 5, 99, augment).draw_samples()[0])


def test_intensity_draws_follow_each_sample(subjects):
    pp = _pp()
    _, subs = subjects
    v = _bare_source(subs, 4, 7, True, intensity=True)
    mats, ab = v.draw_samples()
    rng = np.random.RandomState(7)
    for i in range(4):
        s = int(rng.randint(len(subs)))
        j, T = subs[s].draw(rng, True)
        assert np.array_equal(mats[i], subs[s].matrices((j - 1, j, j + 1), T, v.offsets[s]))
        a, b = rng.uniform(*pp.CONTRAST_RANGE), rng.uniform(*pp.OFFSET_RANGE)
        assert ab[i, 0] == np.float32(a) and ab[i, 1] == np.float32(b)
        assert 0.75 <= ab[i, 0] <= 1.25 and -0.1 <= ab[i, 1] <= 0.1
    assert ab.dtype == np.float32 and ab.shape == (4, 2)


def test_command_line_flags_are_rejected_where_they_do_not_apply(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import prepare_data, train_segmenter, train_gan
    pairs = tmp_path / "pairs"
    pairs.write_text("")
    base = ["--modality", "ct", "--pairs", str(pairs), "--out", str(tmp_path / "out")]
    for extra in (["--split", "train", "--no-augment", "--elastic"], ["--split", "val", "--intensity"],
                  ["--split", "test", "--elastic", "--intensity"]):
        with pytest.raises(SystemExit):
            prepare_data.main(base + extra)
    with pytest.raises(ValueError):
        prepare_data.prepare("ct", [], "val", str(tmp_path / "out2"), elastic=True)
    for flag in ("--elastic", "--intensity"):
        with pytest.raises(SystemExit):
            train_segmenter.main([flag, "--synthetic"])
        with pytest.raises(SystemExit):
            train_gan.main("train-gan", ["--phase", "train-gan", flag, "--synthetic"])
