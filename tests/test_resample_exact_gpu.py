"""pnp_resample_planes (csrc/resample.cu) bit for bit against its numpy restatement oracle/resample_exact.py, at the C-ABI:
random, rotated, scaled and out-of-volume matrices, odd volume sizes and an axis of length 1, label_planes 0, 1 and C with and
without the image, NaN-sentinel outputs, the grid-stride cap with several iterations and a single partial CTA; every rejected
argument leaves its outputs untouched; repeated calls are bit-identical.  The case table is shared with
tests/test_resample_exact_cpu.py, which checks the restatement itself."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import resample_exact as R
from tests.cabi import BAD_ARG, UNSUPPORTED, assert_bits, assert_untouched, lib, sentinel, snapshot, sync

F32 = np.float32
LAB_SENTINEL = -0x5EED

# (tag, volume shape, B, H, W, C, image, label_planes)
CASES = [
    ("odd", (9, 13, 7), 2, 11, 17, 3, True, 1),
    ("odd_all_planes", (9, 13, 7), 2, 11, 17, 3, True, 3),
    ("no_labels", (5, 6, 11), 3, 9, 8, 4, True, 0),
    ("labels_only_middle", (12, 8, 10), 2, 16, 9, 5, False, 1),
    ("labels_only_all", (12, 8, 10), 1, 10, 13, 5, False, 5),
    ("unit_axis", (1, 15, 9), 2, 13, 12, 3, True, 3),
    ("unit_axes", (7, 1, 1), 1, 6, 5, 2, True, 2),
    ("one_plane", (6, 6, 6), 3, 7, 7, 1, True, 1),
    ("partial_cta", (8, 9, 10), 1, 5, 7, 3, True, 3),
    ("slices_as_channels", (40, 44, 33), 1, 64, 64, 21, True, 21),
    ("cap", (37, 41, 29), 2, 256, 256, 70, True, 1),
]
KINDS = ("random", "rotated", "scaled", "outside", "halfint", "identity")


def operands(case):
    """(vol fp32, cls uint8, mats fp32 [B, C, 3, 3]) of a case, drawn on the host from a seed of the case; each plane's matrix
    is one of KINDS in turn"""
    tag, shape, B, H, W, C, image, lp = case
    rng = np.random.RandomState(sum(map(ord, tag)))
    n = np.array(shape, np.float64)
    vol = rng.standard_normal(shape).astype(F32) * F32(3)
    cls = rng.randint(0, 8, shape).astype(np.uint8)
    mats = np.zeros((B * C, 3, 3))
    for p in range(B * C):
        kind = KINDS[(p + len(tag)) % len(KINDS)]
        if kind == "identity":
            m = np.array([[1.0, 0, 0], [0, 1.0, 0], [0, 0, p % shape[2]]])
        elif kind == "halfint":      # coordinates on half-integers: label ties
            m = np.array([[1.0, 0, -0.5], [0, 0.5, 0.5], [0, 0, rng.randint(0, shape[2]) + 0.5]])
        elif kind == "outside":
            m = np.array([[1.5, 0.2, -0.6 * n[0]], [0.1, 1.5, -0.5 * n[1]], [0.3, -0.2, rng.uniform(-2, 2) * n[2]]])
        elif kind == "scaled":
            m = np.diag([rng.uniform(0.3, 2.5) * n[0] / H, rng.uniform(0.3, 2.5) * n[1] / W, 1.0])
            m[2] = [0, 0, rng.uniform(0, n[2] - 1)]
            m[:2, 2] = rng.uniform(-1, 2, 2)
        elif kind == "rotated":
            th = rng.uniform(-np.pi, np.pi)
            sr, sc = n[0] / H, n[1] / W
            m = np.array([[np.cos(th) * sr, -np.sin(th) * sc, 0], [np.sin(th) * sr, np.cos(th) * sc, 0], [0, 0, rng.uniform(0, n[2] - 1)]])
            m[0, 2] = (n[0] - 1) / 2 - m[0, 0] * (H - 1) / 2 - m[0, 1] * (W - 1) / 2
            m[1, 2] = (n[1] - 1) / 2 - m[1, 0] * (H - 1) / 2 - m[1, 1] * (W - 1) / 2
        else:
            m = rng.uniform(-1.5, 1.5, (3, 3)) * np.array([n[0] / H, n[1] / W, 1.0])[:, None]
            m[:, 2] = rng.uniform(-2, n + 1)
        mats[p] = m
    return vol, cls, mats.astype(F32).reshape(B, C, 3, 3)


def _call(_C, rt, vol, cls, dims, mats, B, H, W, C, img, lab, lp):
    return _C.lib.pnp_resample_planes(None if vol is None else vol.data_ptr(), None if cls is None else cls.data_ptr(), *dims,
                                      None if mats is None else mats.data_ptr(), B, H, W, C, None if img is None else img.data_ptr(),
                                      None if lab is None else lab.data_ptr(), lp, rt.stream())


def _buffers(B, H, W, C, image, lp):
    img = sentinel((B, H, W, C)) if image else None
    lab = None
    if lp:
        lab = torch.full((B, H, W) if lp == 1 else (B, H, W, C), LAB_SENTINEL, dtype=torch.int64, device="cuda")
    return img, lab


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_pnp_resample_planes_bit_exact(case):
    _C, rt = lib()
    tag, shape, B, H, W, C, image, lp = case
    vol, cls, mats = operands(case)
    dv, dc, dm = (torch.from_numpy(a).cuda() for a in (vol, cls, mats))
    img, lab = _buffers(B, H, W, C, image, lp)
    spare = torch.full((B, H, W), LAB_SENTINEL, dtype=torch.int64, device="cuda") if not lp else None
    assert _call(_C, rt, dv, dc, shape, dm, B, H, W, C, img, spare if not lp else lab, lp) == 0
    sync()
    ref_img, ref_lab = R.resample_ref(vol, cls, mats, B, H, W, C, lp, image)
    if image:
        assert_bits(tag + " image", img, torch.from_numpy(ref_img).cuda())
    if lp:
        assert torch.equal(lab.cpu(), torch.from_numpy(ref_lab)), tag + " labels"
    else:
        assert bool((spare == LAB_SENTINEL).all()), "label_planes = 0 wrote the label buffer"
    # repeated calls are bit-identical
    if image:
        first = img.clone()
        assert _call(_C, rt, dv, dc, shape, dm, B, H, W, C, img, lab, lp) == 0
        sync()
        assert torch.equal(first.view(torch.int32), img.view(torch.int32))


@pytest.mark.gpu
def test_functional_wrapper_equals_the_c_abi():
    _C, rt = lib()
    from pnp_b200 import functional as F
    case = CASES[1]
    tag, shape, B, H, W, C, image, lp = case
    vol, cls, mats = operands(case)
    dv, dc, dm = (torch.from_numpy(a).cuda() for a in (vol, cls, mats))
    img, lab = F.resample_planes(dv, dc, dm, H, W, True, C)
    mid_img, mid = F.resample_planes(None, dc, dm, H, W, False, 1)
    sync()
    ref_img, ref_lab = R.resample_ref(vol, cls, mats, B, H, W, C, C)
    assert_bits("functional image", img, torch.from_numpy(ref_img).cuda())
    assert torch.equal(lab.cpu(), torch.from_numpy(ref_lab)) and mid_img is None
    assert torch.equal(mid.cpu(), torch.from_numpy(ref_lab[..., C // 2]))


@pytest.mark.gpu
def test_rejected_arguments_leave_the_outputs_untouched():
    _C, rt = lib()
    B, H, W, C = 2, 5, 6, 3
    shape = (4, 5, 6)
    vol = torch.randn(shape, device="cuda")
    cls = torch.randint(0, 5, shape, dtype=torch.uint8, device="cuda")
    mats = torch.randn(B, C, 3, 3, device="cuda")
    img, lab = _buffers(B, H, W, C, True, C)
    bufs = {"img": img, "lab": lab}
    before = snapshot(bufs)
    big = 1 << 23
    bad = [
        ("NULL mats", BAD_ARG, (vol, cls, shape, None, B, H, W, C, img, lab, C)),
        ("NULL vol with an image", BAD_ARG, (None, cls, shape, mats, B, H, W, C, img, lab, C)),
        ("NULL cls with labels", BAD_ARG, (vol, None, shape, mats, B, H, W, C, img, lab, C)),
        ("NULL lab with labels", BAD_ARG, (vol, cls, shape, mats, B, H, W, C, img, None, C)),
        ("no output", BAD_ARG, (vol, cls, shape, mats, B, H, W, C, None, lab, 0)),
        ("n0 = 0", BAD_ARG, (vol, cls, (0, 5, 6), mats, B, H, W, C, img, lab, C)),
        ("n2 < 0", BAD_ARG, (vol, cls, (4, 5, -6), mats, B, H, W, C, img, lab, C)),
        ("B = 0", BAD_ARG, (vol, cls, shape, mats, 0, H, W, C, img, lab, C)),
        ("H < 0", BAD_ARG, (vol, cls, shape, mats, B, -5, W, C, img, lab, C)),
        ("W = 0", BAD_ARG, (vol, cls, shape, mats, B, H, 0, C, img, lab, C)),
        ("C = 0", BAD_ARG, (vol, cls, shape, mats, B, H, W, 0, img, lab, 0)),
        ("label_planes = 2 with C = 3", UNSUPPORTED, (vol, cls, shape, mats, B, H, W, C, img, lab, 2)),
        ("label_planes = -1", UNSUPPORTED, (vol, cls, shape, mats, B, H, W, C, img, lab, -1)),
        ("n1 above PNP_RS_MAX_DIM", UNSUPPORTED, (vol, cls, (1, big + 1, 1), mats, B, H, W, C, img, lab, C)),
        ("W above PNP_RS_MAX_DIM", UNSUPPORTED, (vol, cls, shape, mats, 1, 1, big + 1, 1, img, lab, 1)),
        ("n0 n1 n2 = 2^31", UNSUPPORTED, (vol, cls, (1 << 11, 1 << 10, 1 << 10), mats, B, H, W, C, img, lab, C)),
        ("B H W C = 2^31", UNSUPPORTED, (vol, cls, shape, mats, 1 << 7, 1 << 10, 1 << 10, 1 << 4, img, lab, 1)),
        ("B C 9 >= 2^31", UNSUPPORTED, (vol, cls, shape, mats, 1 << 13, 1, 1, 1 << 15, None, lab, 1)),
    ]
    for what, rc_want, args in bad:
        rc = _call(_C, rt, *args)
        assert rc == rc_want, (what, rc)
        assert_untouched(what, "pnp_resample_planes", bufs, before)
    msg = _C.lib.pnp_error_string(BAD_ARG)
    assert isinstance(msg, bytes) and msg
    assert ctypes.c_int(_C.lib.pnp_version()).value >= 103
