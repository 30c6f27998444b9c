"""The opt-in elastic and intensity augmentations on the device, bit for bit against oracle/augment_exact.py:
* pnp_smooth_noise_field at K = 1 and 2, R = 0, R >= W / 2, the largest R, sizes off the tiles, partial CTAs and grid-stride sweeps
  of both passes;
* pnp_resample_planes_aug with disp, gain and ab alone and together, at label_planes 0, 1 and C; a zero field with a = 1, b = 0
  equals pnp_resample_planes as values; rejected arguments of both calls leave their outputs untouched;
* data.VolumeSource with the flags on equals the oracle fed the same matrices, seeds and draws, and with them off is
  bit-identical to a twin drawn through plain resample_planes;
* prepare_data --elastic --intensity records equal the kernel's output; both trainers run a few steps on augmented streams."""
import os

import numpy as np
import pytest
import torch

from oracle import augment_exact as A
from oracle.elementwise_exact import NUM_SMS
from tests.cabi import BAD_ARG, UNSUPPORTED, assert_bits, assert_untouched, lib, sentinel, snapshot, sync
from tests import mmwhs_phantom as ph

pytestmark = pytest.mark.gpu
F32 = np.float32
CAP = NUM_SMS * 64

# (tag, B, K, H, W, sigma): pass-1 tiles B K H ceil(W / 256), pass-2 tiles B K ceil(H / 64) ceil(W / 32), capped at CAP CTAs
FIELD_CASES = [
    ("r0", 2, 1, 7, 9, 0.1),
    ("r_over_half_w", 1, 2, 13, 6, 2.0),
    ("partial_tiles", 2, 2, 70, 37, 3.0),
    ("elastic", 3, 2, 256, 256, 10.0),
    ("bias_max_r", 2, 1, 256, 256, 32.0),
    ("max_r_small_plane", 1, 1, 40, 300, 32.0),
    ("sweeps", 17, 2, 70, 4000, 0.7),
    ("one_row", 1, 1, 1, 30, 1.5),
]


def _tiles(B, K, H, W):
    return B * K * H * -(-W // 256), B * K * -(-H // 64) * -(-W // 32)


def test_field_cases_cover_the_launch_regimes():
    t1 = [_tiles(*c[1:5])[0] for c in FIELD_CASES]
    t2 = [_tiles(*c[1:5])[1] for c in FIELD_CASES]
    assert max(t1) > CAP and max(t2) > CAP                         # grid-stride sweeps in both passes
    assert min(t1) == 1 and min(t2) == 1                           # a single partial CTA
    assert any(len(A.gaussian_taps(c[5])) == 1 for c in FIELD_CASES)
    assert any((len(A.gaussian_taps(c[5])) - 1) // 2 >= c[4] / 2 for c in FIELD_CASES)
    assert any((len(A.gaussian_taps(c[5])) - 1) // 2 == A.NF_MAX_R for c in FIELD_CASES)


def _field_call(_C, rt, seed, stream, B, K, H, W, taps, R, amp, lo, hi, out, tmp):
    return _C.lib.pnp_smooth_noise_field(seed, stream, B, K, H, W, None if taps is None else taps.data_ptr(), R, amp, lo, hi,
                                         None if out is None else out.data_ptr(), None if tmp is None else tmp.data_ptr(), rt.stream())


@pytest.mark.parametrize("case", FIELD_CASES, ids=lambda c: c[0])
def test_smooth_noise_field_bit_exact(case):
    _C, rt = lib()
    tag, B, K, H, W, sigma = case
    taps = A.gaussian_taps(sigma)
    R = (len(taps) - 1) // 2
    seed, stream = 0xC0FFEE + len(tag), (0xE1A5 << 32) | len(tag)
    amp, lo, hi = (160.0, -16.0, 16.0) if K == 2 else (20.0, -0.5, 0.5)
    dt = torch.from_numpy(taps).cuda()
    out, tmp = sentinel((B, K, H, W)), sentinel((B, K, H, W))
    assert _field_call(_C, rt, seed, stream, B, K, H, W, dt, R, amp, lo, hi, out, tmp) == 0
    sync()
    ref = A.noise_field(seed, stream, B, K, H, W, taps, amp, lo, hi)
    assert_bits(tag, out, torch.from_numpy(ref).cuda())
    assert_bits(tag + " pass 1", tmp, torch.from_numpy(A.smooth_pass(A.uniforms(seed, stream, B, K, H, W), taps, -1)).cuda())
    first = out.clone()
    assert _field_call(_C, rt, seed, stream, B, K, H, W, dt, R, amp, lo, hi, out, tmp) == 0
    sync()
    assert torch.equal(first.view(torch.int32), out.view(torch.int32))


def test_functional_smooth_noise_field_equals_the_oracle():
    lib()
    from pnp_b200 import functional as F
    taps = A.gaussian_taps(10.0)
    out = F.smooth_noise_field(5, 7, 2, 2, 64, 48, torch.from_numpy(taps).cuda(), 160.0, -16.0, 16.0)
    sync()
    assert_bits("functional", out, torch.from_numpy(A.noise_field(5, 7, 2, 2, 64, 48, taps, 160.0, -16.0, 16.0)).cuda())


def _fields(B, H, W, seed, kinds):
    """(disp, gain, ab) of a case, fp32 host arrays or None: large displacements (samples leave the volume), gains in [0.5, 1.5]"""
    rng = np.random.RandomState(seed)
    disp = (rng.standard_normal((B, 2, H, W)) * 3).astype(F32) if "disp" in kinds else None
    gain = rng.uniform(-0.5, 0.5, (B, H, W)).astype(F32) if "gain" in kinds else None
    ab = np.stack([rng.uniform(0.75, 1.25, B), rng.uniform(-0.1, 0.1, B)], 1).astype(F32) if "ab" in kinds else None
    return disp, gain, ab


def _aug_call(_C, rt, vol, cls, dims, mats, B, H, W, C, img, lab, lp, disp, gain, ab):
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    return _C.lib.pnp_resample_planes_aug(p(vol), p(cls), *dims, p(mats), B, H, W, C, p(img), p(lab), lp, p(disp), p(gain), p(ab),
                                          rt.stream())


LAB_SENTINEL = -0x5EED
# (tag, volume shape, B, H, W, C, image, label_planes)
AUG_CASES = [
    ("odd", (9, 13, 7), 2, 11, 17, 3, True, 1),
    ("odd_all_planes", (9, 13, 7), 2, 11, 17, 3, True, 3),
    ("no_labels", (5, 6, 11), 3, 9, 8, 4, True, 0),
    ("labels_only_all", (12, 8, 10), 1, 10, 13, 5, False, 5),
    ("unit_axis", (1, 15, 9), 2, 13, 12, 3, True, 3),
    ("partial_cta", (8, 9, 10), 1, 5, 7, 3, True, 3),
    ("cap", (37, 41, 29), 2, 256, 256, 70, True, 1),
]


def operands(case):
    """(vol fp32, cls uint8, mats fp32 [B, C, 3, 3]) of a case: plane p samples a rotated and scaled copy of the volume's slice
    p mod n0, some planes partly outside it"""
    tag, shape, B, H, W, C, image, lp = case
    rng = np.random.RandomState(sum(map(ord, tag)))
    n = np.array(shape, np.float64)
    vol = rng.standard_normal(shape).astype(F32) * F32(3)
    cls = rng.randint(0, 8, shape).astype(np.uint8)
    mats = np.zeros((B * C, 3, 3))
    for p in range(B * C):
        th, sc = rng.uniform(-np.pi, np.pi), rng.uniform(0.5, 1.6)
        sr, scc = sc * n[1] / H, sc * n[2] / W
        m = np.array([[0, 0, rng.uniform(-0.5, n[0] - 0.5)], [np.cos(th) * sr, -np.sin(th) * scc, 0], [np.sin(th) * sr, np.cos(th) * scc, 0]])
        m[1, 2] = (n[1] - 1) / 2 - m[1, 0] * (H - 1) / 2 - m[1, 1] * (W - 1) / 2 + rng.uniform(-2, 2)
        m[2, 2] = (n[2] - 1) / 2 - m[2, 0] * (H - 1) / 2 - m[2, 1] * (W - 1) / 2 + rng.uniform(-2, 2)
        mats[p] = m
    return vol, cls, mats.astype(F32).reshape(B, C, 3, 3)


KINDS = [("disp",), ("gain",), ("ab",), ("disp", "gain", "ab")]


@pytest.mark.parametrize("kinds", KINDS, ids=lambda k: "+".join(k))
@pytest.mark.parametrize("case", AUG_CASES, ids=lambda c: c[0])
def test_resample_planes_aug_bit_exact(case, kinds):
    _C, rt = lib()
    tag, shape, B, H, W, C, image, lp = case
    if not image and kinds != ("disp",):
        pytest.skip("gain and ab act on the image only")
    vol, cls, mats = operands(case)
    disp, gain, ab = _fields(B, H, W, len(tag) + len(kinds), kinds)
    dv, dc, dm = (torch.from_numpy(a).cuda() for a in (vol, cls, mats))
    dd, dg, dab = (None if a is None else torch.from_numpy(a).cuda() for a in (disp, gain, ab))
    img = sentinel((B, H, W, C)) if image else None
    lab = torch.full((B, H, W) if lp <= 1 else (B, H, W, C), LAB_SENTINEL, dtype=torch.int64, device="cuda")
    assert _aug_call(_C, rt, dv, dc, shape, dm, B, H, W, C, img, lab, lp, dd, dg, dab) == 0
    sync()
    ref_img, ref_lab = A.resample_aug_ref(vol, cls, mats, B, H, W, C, lp, image, disp, gain, ab)
    if image:
        assert_bits(tag + " image", img, torch.from_numpy(ref_img).cuda())
    if lp:
        assert torch.equal(lab.cpu(), torch.from_numpy(ref_lab)), tag + " labels"
    else:
        assert bool((lab == LAB_SENTINEL).all())


@pytest.mark.parametrize("case", AUG_CASES, ids=lambda c: c[0])
def test_zero_fields_equal_resample_planes(case):
    _C, rt = lib()
    tag, shape, B, H, W, C, image, lp = case
    vol, cls, mats = operands(case)
    dv, dc, dm = (torch.from_numpy(a).cuda() for a in (vol, cls, mats))
    zd, zg = torch.zeros(B, 2, H, W, device="cuda"), torch.zeros(B, H, W, device="cuda")
    ab = torch.tensor([[1.0, 0.0]] * B, device="cuda")
    outs = []
    for aug in (False, True):
        img = sentinel((B, H, W, C)) if image else None
        lab = torch.full((B, H, W) if lp <= 1 else (B, H, W, C), LAB_SENTINEL, dtype=torch.int64, device="cuda") if lp else None
        if aug:
            assert _aug_call(_C, rt, dv, dc, shape, dm, B, H, W, C, img, lab, lp, zd, zg if image else None, ab if image else None) == 0
        else:
            assert _C.lib.pnp_resample_planes(dv.data_ptr(), dc.data_ptr(), *shape, dm.data_ptr(), B, H, W, C,
                                              None if img is None else img.data_ptr(), None if lab is None else lab.data_ptr(), lp,
                                              rt.stream()) == 0
        outs.append((img, lab))
    sync()
    if image:
        assert torch.equal(outs[0][0], outs[1][0])                  # as values: a * v + 0 turns -0 into +0
    if lp:
        assert torch.equal(outs[0][1], outs[1][1])
    # all three NULL: the <true> kernel without fields is bit-identical
    if image:
        img = sentinel((B, H, W, C))
        assert _aug_call(_C, rt, dv, dc, shape, dm, B, H, W, C, img, outs[1][1], lp, None, None, None) == 0
        sync()
        assert torch.equal(img.view(torch.int32), outs[0][0].view(torch.int32))


def test_rejected_arguments_leave_the_outputs_untouched():
    _C, rt = lib()
    B, H, W, C = 2, 5, 6, 3
    shape = (4, 5, 6)
    vol = torch.randn(shape, device="cuda")
    cls = torch.randint(0, 5, shape, dtype=torch.uint8, device="cuda")
    mats = torch.randn(B, C, 3, 3, device="cuda")
    disp, gain, ab = torch.zeros(B, 2, H, W, device="cuda"), torch.zeros(B, H, W, device="cuda"), torch.ones(B, 2, device="cuda")
    img = sentinel((B, H, W, C))
    lab = torch.full((B, H, W, C), LAB_SENTINEL, dtype=torch.int64, device="cuda")
    bufs = {"img": img, "lab": lab}
    before = snapshot(bufs)
    bad = [
        ("NULL mats", BAD_ARG, (vol, cls, shape, None, B, H, W, C, img, lab, C, disp, gain, ab)),
        ("no output", BAD_ARG, (vol, cls, shape, mats, B, H, W, C, None, lab, 0, disp, None, None)),
        ("gain without img", BAD_ARG, (None, cls, shape, mats, B, H, W, C, None, lab, C, disp, gain, None)),
        ("ab without img", BAD_ARG, (None, cls, shape, mats, B, H, W, C, None, lab, C, None, None, ab)),
        ("NULL lab with labels", BAD_ARG, (vol, cls, shape, mats, B, H, W, C, img, None, C, disp, gain, ab)),
        ("W = 0", BAD_ARG, (vol, cls, shape, mats, B, H, 0, C, img, lab, C, disp, gain, ab)),
        ("label_planes = 2", UNSUPPORTED, (vol, cls, shape, mats, B, H, W, C, img, lab, 2, disp, gain, ab)),
        ("B 2 H W = 2^31 with disp", UNSUPPORTED, (None, cls, shape, mats, 1 << 10, 1 << 10, 1 << 10, 1, None, lab, 1, disp, None,
                                                   None)),
    ]
    for what, want, args in bad:
        assert _aug_call(_C, rt, *args) == want, what
        assert_untouched(what, "pnp_resample_planes_aug", bufs, before)

    taps = torch.from_numpy(A.gaussian_taps(2.0)).cuda()
    big = torch.from_numpy(A.gaussian_taps(40.0)).cuda()
    out, tmp = sentinel((B, 2, H, W)), sentinel((B, 2, H, W))
    fb = {"out": out, "tmp": tmp}
    fbefore = snapshot(fb)
    nan = float("nan")
    fbad = [
        ("NULL taps", BAD_ARG, (1, 2, B, 2, H, W, None, 8, 1.0, -1.0, 1.0, out, tmp)),
        ("NULL out", BAD_ARG, (1, 2, B, 2, H, W, taps, 8, 1.0, -1.0, 1.0, None, tmp)),
        ("NULL tmp", BAD_ARG, (1, 2, B, 2, H, W, taps, 8, 1.0, -1.0, 1.0, out, None)),
        ("out == tmp", BAD_ARG, (1, 2, B, 2, H, W, taps, 8, 1.0, -1.0, 1.0, out, out)),
        ("K = 0", BAD_ARG, (1, 2, B, 0, H, W, taps, 8, 1.0, -1.0, 1.0, out, tmp)),
        ("H < 0", BAD_ARG, (1, 2, B, 2, -H, W, taps, 8, 1.0, -1.0, 1.0, out, tmp)),
        ("R < 0", BAD_ARG, (1, 2, B, 2, H, W, taps, -1, 1.0, -1.0, 1.0, out, tmp)),
        ("lo > hi", BAD_ARG, (1, 2, B, 2, H, W, taps, 8, 1.0, 1.0, -1.0, out, tmp)),
        ("NaN lo", BAD_ARG, (1, 2, B, 2, H, W, taps, 8, 1.0, nan, 1.0, out, tmp)),
        ("NaN amp", BAD_ARG, (1, 2, B, 2, H, W, taps, 8, nan, -1.0, 1.0, out, tmp)),
        ("R above PNP_NF_MAX_R", UNSUPPORTED, (1, 2, B, 2, H, W, big, 160, 1.0, -1.0, 1.0, out, tmp)),
        ("B K H W = 2^31", UNSUPPORTED, (1, 2, 1 << 8, 2, 1 << 11, 1 << 11, taps, 8, 1.0, -1.0, 1.0, out, tmp)),
    ]
    for what, want, args in fbad:
        assert _field_call(_C, rt, *args) == want, what
        assert_untouched(what, "pnp_smooth_noise_field", fb, fbefore)


# ------------------------------------------------------------------------------------------------------------------------------
# host layer: VolumeSource, prepare_data, the trainers
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def phantoms(tmp_path_factory):
    d = tmp_path_factory.mktemp("aug_gpu")
    src = d / "raw"
    src.mkdir()
    train = ph.write_pairs(str(src), "ct", [41, 42])
    val = ph.write_pairs(str(src), "mr", [43], spacing=(1.1, 0.7, 1.3))
    return {"dir": d, "train": train, "val": val}


def _oracle_batch(vs, mats, ab, t):
    """the oracle's batch of a VolumeSource draw: its matrices and (a, b), the fields of draw t of its seed"""
    from pnp_b200 import preprocess as pp
    B, S = vs.B, pp.SIZE
    disp = gain = None
    if vs.elastic:
        disp = A.noise_field(vs.seed, pp.field_stream(pp.ELASTIC_STREAM_TAG, t), B, 2, S, S, A.gaussian_taps(pp.ELASTIC_SIGMA),
                             pp.ELASTIC_ALPHA, -pp.ELASTIC_MAX_PX, pp.ELASTIC_MAX_PX)
    if vs.intensity:
        gain = A.noise_field(vs.seed, pp.field_stream(pp.BIAS_STREAM_TAG, t), B, 1, S, S, A.gaussian_taps(pp.BIAS_SIGMA),
                             pp.BIAS_BETA, -pp.BIAS_MAX, pp.BIAS_MAX)[:, 0]
    return A.resample_aug_ref(vs.vol.cpu().numpy(), vs.cls.cpu().numpy(), mats, B, S, S, 3, 1, True, disp, gain, ab)


@pytest.mark.parametrize("flags", [(True, False), (False, True), (True, True)], ids=["elastic", "intensity", "both"])
def test_volume_source_with_flags_equals_the_oracle(phantoms, flags):
    lib()
    from pnp_b200.data import VolumeSource
    elastic, intensity = flags
    B = 3
    vs = VolumeSource(phantoms["train"], B, 1234, elastic=elastic, intensity=intensity)
    twin = VolumeSource(phantoms["train"], B, 1234, elastic=elastic, intensity=intensity)   # replays the generator's draws
    for t in range(3):
        x, y = vs.next()
        mats, ab = twin.draw_samples()
        sync()
        ref_img, ref_lab = _oracle_batch(vs, mats, ab, t)
        assert_bits("VolumeSource draw %d" % t, x, torch.from_numpy(ref_img).cuda())
        assert torch.equal(y.cpu(), torch.from_numpy(ref_lab)), t
        assert bool(torch.isfinite(x).all())
    assert vs.draws == 3


def test_volume_source_flags_off_is_bit_identical_to_plain_resampling(phantoms):
    lib()
    from pnp_b200.data import VolumeSource
    from pnp_b200 import functional as F
    B = 4
    vs = VolumeSource(phantoms["train"], B, 99)
    twin = VolumeSource(phantoms["train"], B, 99)
    assert not hasattr(vs, "_tmp") and vs._fields == [{}, {}]
    from pnp_b200 import _C
    for _ in range(3):
        n0 = _C.launch_count
        x, y = vs.next()
        assert _C.launch_count - n0 == 1                            # one launch, no field calls
        m = torch.from_numpy(twin.draw_matrices()).cuda()
        img, lab = F.resample_planes(twin.vol, twin.cls, m, 256, 256, True, 1)
        sync()
        assert torch.equal(x.view(torch.int32), img.view(torch.int32)) and torch.equal(y, lab)
    assert vs.rng.randint(1 << 30) == twin.rng.randint(1 << 30)
    both = VolumeSource(phantoms["train"], B, 99, elastic=True, intensity=True)
    n0 = _C.launch_count
    both.next()
    assert _C.launch_count - n0 == 3                                # two field calls and the resampling
    with pytest.raises(ValueError):
        VolumeSource(phantoms["train"], B, 99, augment=False, elastic=True)


def test_prepare_data_elastic_intensity_records_equal_the_kernel(phantoms):
    lib()
    from pnp_b200 import prepare_data, preprocess as pp, functional as F, tfrecord
    spv = 5
    d = phantoms["dir"]
    pf = str(d / "train_pairs")
    with open(pf, "w") as f:
        f.write("".join("%s %s\n" % p for p in phantoms["train"]))
    out = str(d / "out")
    prepare_data.main(["--modality", "ct", "--pairs", pf, "--split", "train", "--out", out, "--slices-per-volume", str(spv),
                       "--seed", "6", "--elastic", "--intensity"])
    files = [ln.strip() for ln in open(os.path.join(out, "lists", "ct_train_list")) if ln.strip()]
    assert len(files) == spv * len(phantoms["train"])
    rng = np.random.RandomState(6)
    taps_e = torch.from_numpy(pp.gaussian_taps(pp.ELASTIC_SIGMA)).cuda()
    taps_b = torch.from_numpy(pp.gaussian_taps(pp.BIAS_SIGMA)).cuda()
    k = 0
    for t, (im, lb) in enumerate(phantoms["train"]):        # one launch per subject (spv <= CHUNK): draw t is the subject
        s = pp.Subject(im, lb, reach_px=pp.ELASTIC_REACH_PX)
        draws = []
        for _ in range(spv):
            j, T = s.draw(rng, True)
            draws.append((j, T, pp.intensity_draw(rng)))
        mats = np.stack([s.matrices((j - 1, j, j + 1), T) for j, T, _ in draws])
        ab = np.asarray([d_[2] for d_ in draws], np.float64).astype(F32)
        vol, cls = torch.from_numpy(s.vol).cuda(), torch.from_numpy(s.cls).cuda()
        disp = F.smooth_noise_field(6, pp.field_stream(pp.ELASTIC_STREAM_TAG, t), spv, 2, 256, 256, taps_e, pp.ELASTIC_ALPHA,
                                    -pp.ELASTIC_MAX_PX, pp.ELASTIC_MAX_PX)
        gain = F.smooth_noise_field(6, pp.field_stream(pp.BIAS_STREAM_TAG, t), spv, 1, 256, 256, taps_b, pp.BIAS_BETA, -pp.BIAS_MAX,
                                    pp.BIAS_MAX)[:, 0]
        img, lab = F.resample_planes(vol, cls, torch.from_numpy(mats).cuda(), 256, 256, True, 3, disp=disp, gain=gain,
                                     ab=torch.from_numpy(ab).cuda())
        sync()
        ref_img, ref_lab = A.resample_aug_ref(s.vol, s.cls, mats, spv, 256, 256, 3, 3, True, disp.cpu().numpy(),
                                              gain.cpu().numpy(), ab)
        assert np.array_equal(img.cpu().numpy().view(np.int32), ref_img.view(np.int32))
        assert np.array_equal(lab.cpu().numpy(), ref_lab)
        img, lab = img.cpu().numpy(), lab.cpu().numpy()
        for i in range(spv):
            ex = tfrecord.parse_example(next(tfrecord.read_records(files[k])))
            k += 1
            assert np.array_equal(np.frombuffer(ex["data_vol"], "<f4").reshape(256, 256, 3).view(np.int32), img[i].view(np.int32))
            assert np.array_equal(np.frombuffer(ex["label_vol"], "<f4").reshape(256, 256, 3), lab[i].astype(np.float32))


def test_both_trainers_run_with_the_flags(phantoms, tmp_path, monkeypatch):
    """the entry points with --elastic --intensity: a few steps of each trainer on phantom volumes, augmented training streams
    and plain validation streams"""
    lib()
    from pnp_b200 import train_segmenter, train_gan, runtime as rt, data
    rt.set_conv_backend("auto")
    made = []
    real = data.VolumeSource

    class Spy(real):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            made.append((self.elastic, self.intensity))

    monkeypatch.setattr(data, "VolumeSource", Spy)
    train, val = phantoms["train"], phantoms["val"]
    lists = tmp_path / "lists"
    lists.mkdir()
    for name, pairs in (("mr_train_volumes", val), ("mr_val_volumes", val), ("ct_train_volumes", train), ("ct_val_volumes", train)):
        (lists / name).write_text("".join("%s %s\n" % p for p in pairs))
    monkeypatch.chdir(tmp_path)
    train_segmenter.main(["--batch-size", "2", "--training-iters", "2", "--epochs", "1", "--synthetic", "--train-volumes",
                          str(lists / "ct_train_volumes"), "--val-volumes", str(lists / "ct_val_volumes"), "--elastic",
                          "--intensity", "--output-path", str(tmp_path / "seg")])
    assert made == [(True, True), (False, False)]
    made.clear()
    import pnp_b200.train_gan as tg
    monkeypatch.setitem(tg.train_config, "dis_sub_iter", 1)
    train_gan.main("train-gan", ["--phase", "train-gan", "--batch-size", "2", "--training-iters", "2", "--epochs", "1",
                                 "--synthetic", "--lists", str(lists), "--volumes", "--elastic", "--intensity"])
    assert made == [(True, True), (True, True), (False, False), (False, False)]
    assert all(bool(torch.isfinite(v).all()) for v in rt.global_variables())
