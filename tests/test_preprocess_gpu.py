"""The data preparation end to end on seeded phantom subjects (tests/mmwhs_phantom.py: ellipsoids carrying all seven MMWHS values,
anisotropic spacing, permuted and flipped affines written with nifti.save):
* prepare_data for train (augmented), val (--no-augment) and test; the records read back through TFRecordSource(num_threads=0)
  are bit-equal to pnp_resample_planes' output for the same draws, all three label planes included;
* each test volume, after test_eval's flips, is bit-equal to the unaugmented training slices at the same positions, and its
  affine is the subject's;
* VolumeSource: the same seed gives identical batches, the rank seeds different ones; every organ class appears;
* both trainers' train() runs a few iterations on VolumeSource streams with finite losses, and test_eval(..., surface_metrics=True)
  scores the prepared test subjects."""
import os

import numpy as np
import pytest
import torch

from tests import mmwhs_phantom as ph

pytestmark = pytest.mark.gpu
SPV = 6            # augmented samples per training volume


@pytest.fixture(scope="module")
def prepared(tmp_path_factory):
    import pnp_b200  # noqa: F401
    from pnp_b200 import prepare_data
    d = tmp_path_factory.mktemp("mmwhs")
    src = d / "raw"
    src.mkdir()
    train = ph.write_pairs(str(src), "ct", [21, 22], unknown=3)
    val = ph.write_pairs(str(src), "mr", [23], spacing=(1.1, 0.7, 1.3))
    test = ph.write_pairs(str(src), "ct", [24], shape=(40, 36, 30), spacing=(0.9, 1.0, 1.4))
    pf = {}
    for name, pairs in (("train", train), ("val", val), ("test", test)):
        pf[name] = str(d / ("%s_pairs" % name))
        with open(pf[name], "w") as f:
            f.write("".join("%s %s\n" % p for p in pairs))
    out = str(d / "out")
    prepare_data.main(["--modality", "ct", "--pairs", pf["train"], "--split", "train", "--out", out, "--slices-per-volume",
                       str(SPV), "--seed", "5"])
    prepare_data.main(["--modality", "mr", "--pairs", pf["val"], "--split", "val", "--out", out, "--no-augment"])
    prepare_data.main(["--modality", "ct", "--pairs", pf["test"], "--split", "test", "--out", out])
    return {"out": out, "train": train, "val": val, "test": test, "pair_files": pf}


def _lines(path):
    with open(path) as f:
        return [ln.strip() for ln in f if ln.strip()]


def _kernel_samples(pairs, draws_of):
    """pnp_resample_planes' (image, label planes) of every sample, straight from the kernel: [(img [256,256,3], lab [256,256,3])]"""
    from pnp_b200 import preprocess as pp, functional as F
    out = []
    for im, lb in pairs:
        s = pp.Subject(im, lb)
        vol, cls = torch.from_numpy(s.vol).cuda(), torch.from_numpy(s.cls).cuda()
        for j, T in draws_of(s):
            m = torch.from_numpy(s.matrices((j - 1, j, j + 1), T)[None]).cuda()
            img, lab = F.resample_planes(vol, cls, m, 256, 256, True, 3)
            out.append((img[0].cpu().numpy(), lab[0].cpu().numpy()))
    return out


def _check_records(files, expected):
    from pnp_b200 import tfrecord
    assert len(files) == len(expected)
    for f, (img, lab) in zip(files, expected):
        ex = tfrecord.parse_example(next(tfrecord.read_records(f)))
        assert [ex["dsize_dim%d" % i][0] for i in range(3)] == [256, 256, 3]
        assert np.array_equal(np.frombuffer(ex["data_vol"], "<f4").reshape(256, 256, 3).view(np.int32), img.view(np.int32))
        assert np.array_equal(np.frombuffer(ex["label_vol"], "<f4").reshape(256, 256, 3), lab.astype(np.float32))
    src = tfrecord.TFRecordSource(files, len(files), seed=3, num_threads=0)
    x, y = src.next()
    for i, k in enumerate(src.order):
        assert np.array_equal(x[i].numpy().view(np.int32), expected[k][0].view(np.int32))
        assert np.array_equal(y[i].numpy(), expected[k][1][:, :, 1])


def test_records_equal_the_kernel_output(prepared):
    out = prepared["out"]
    train = _lines(os.path.join(out, "lists", "ct_train_list"))
    rng = np.random.RandomState(5)
    _check_records(train, _kernel_samples(prepared["train"], lambda s: [s.draw(rng, True) for _ in range(SPV)]))
    val = _lines(os.path.join(out, "lists", "mr_val_list"))
    _check_records(val, _kernel_samples(prepared["val"], lambda s: [(j, None) for j in range(s.j_lo, s.j_hi + 1)]))
    vols = [ln.split() for ln in _lines(os.path.join(out, "lists", "ct_train_volumes"))]
    assert vols == [[os.path.abspath(a), os.path.abspath(b)] for a, b in prepared["train"]]
    # every organ class appears in the records
    from pnp_b200 import tfrecord
    seen = set()
    for f in train + val:
        seen |= set(np.unique(tfrecord.decode_slice(next(tfrecord.read_records(f)))[1]).tolist())
    assert seen == {0, 1, 2, 3, 4}


def test_test_volumes_equal_the_unaugmented_training_slices(prepared):
    from pnp_b200 import preprocess as pp, nifti
    out = prepared["out"]
    nii = _lines(os.path.join(out, "lists", "ct_test_nii_list"))
    lab = _lines(os.path.join(out, "lists", "ct_test_label_list"))
    assert len(nii) == len(lab) == 1
    s = pp.Subject(*prepared["test"][0])
    vi, vl = nifti.load(nii[0]), nifti.load(lab[0])
    assert vi.shape == vl.shape == (256, 256, s.D)
    assert np.allclose(vi.get_affine(), s.test_affine(), rtol=0, atol=1e-4)
    img = np.flip(np.flip(vi.get_data(), 0), 1)            # test_eval's flip_correction
    cls = np.flip(np.flip(vl.get_data(), 0), 1)
    slices = _kernel_samples(prepared["test"], lambda s: [(j, None) for j in range(s.j_lo, s.j_hi + 1)])
    for j, (im, lb) in zip(range(s.j_lo, s.j_hi + 1), slices):
        assert np.array_equal(np.ascontiguousarray(img[:, :, j - 1:j + 2]).view(np.int32), im.view(np.int32)), j
        assert np.array_equal(cls[:, :, j - 1:j + 2].astype(np.int64), lb), j
    assert set(np.unique(cls).tolist()) == {0, 1, 2, 3, 4}
    # world positions: the stored volume's affine sends each organ's voxels to where the source volume holds them
    src_lab = nifti.load(prepared["test"][0][1])
    lv = np.argwhere(vl.get_data() == 3)
    world = vi.get_affine() @ np.c_[lv, np.ones(len(lv))].T
    vox = np.rint(np.linalg.solve(src_lab.get_affine(), world)[:3]).astype(np.int64)
    ok = np.all((vox >= 0) & (vox < np.array(src_lab.shape)[:, None]), axis=0)
    hit = src_lab.get_data()[tuple(vox[:, ok])] == 500
    assert ok.mean() > 0.99 and hit.mean() > 0.9, (ok.mean(), hit.mean())


def test_volume_source_seeds_and_classes(prepared):
    from pnp_b200.data import VolumeSource
    pairs = prepared["train"]
    a, b, c = VolumeSource(pairs, 4, 1234), VolumeSource(pairs, 4, 1234), VolumeSource(pairs, 4, 1235)
    seen = set()
    for _ in range(3):
        xa, ya = a.next()
        xb, yb = b.next()
        xc, yc = c.next()
        assert xa.is_cuda and xa.shape == (4, 256, 256, 3) and xa.dtype == torch.float32
        assert ya.is_cuda and ya.shape == (4, 256, 256) and ya.dtype == torch.int64
        assert torch.equal(xa.view(torch.int32), xb.view(torch.int32)) and torch.equal(ya, yb)
        assert not torch.equal(xa, xc)
        assert bool(torch.isfinite(xa).all())
        seen |= set(torch.unique(ya).tolist())
    assert seen == {0, 1, 2, 3, 4}
    # a batch stays valid until the next-but-one call
    x1, _ = a.next()
    keep = x1.clone()
    a.next()
    assert torch.equal(x1, keep)
    # unaugmented draws are training slices of the subjects' ranges: each equals a kernel sample with the identity
    u = VolumeSource(pairs[:1], 2, 7, augment=False)
    x, y = u.next()
    from pnp_b200 import preprocess as pp
    s = pp.Subject(*pairs[0])
    rng = np.random.RandomState(7)
    for i in range(2):
        assert rng.randint(1) == 0
        j, T = s.draw(rng, False)
        assert T is None
        (im, lb), = _kernel_samples(pairs[:1], lambda _s: [(j, None)])
        assert np.array_equal(x[i].cpu().numpy().view(np.int32), im.view(np.int32))      # one subject: the stack is its volume
        assert np.array_equal(y[i].cpu().numpy(), lb[:, :, 1])


def test_both_trainers_train_on_volume_sources(prepared, tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv, source_segmenter as seg
    from pnp_b200.data import VolumeSource
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter, init_numpy_params
    rt.set_conv_backend("auto")
    B = 2
    train, val = prepared["train"], prepared["val"]
    out = prepared["out"]
    nii = _lines(os.path.join(out, "lists", "ct_test_nii_list"))
    lab = _lines(os.path.join(out, "lists", "ct_test_label_list"))

    ws, bns = OracleSegmenter.layout()
    snet = seg.Full_DRN(channels=3, n_class=5, batch_size=B,
                        cost_kwargs={"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0})
    rt.load_state_dict(init_numpy_params(ws, bns, 0, 0.05))
    st = seg.Trainer(snet, None, None, num_cls=5, batch_size=B, optimizer="adam", opt_kwargs={"learning_rate": 1e-3},
                     source=VolumeSource(train, B, 1234), val_source=VolumeSource(val, B, 4321), test_nii_list=nii,
                     test_label_list=lab)
    st.train(str(tmp_path / "seg"), training_iters=3, epochs=1, display_step=1, dropout=0.75)
    r = st.val_stats(*st.feed(*VolumeSource(val, B, 9).next()))
    assert np.isfinite(r["loss"]), r
    assert all(bool(torch.isfinite(v).all()) for v in rt.global_variables())
    os.makedirs(str(tmp_path / "seg_test"))
    st.test_eval(str(tmp_path / "seg_test"), surface_metrics=True)
    assert len(st.sample_surface_list) == 1 and (st.sample_surface_list[0]["border_gt"][1:] > 0).all()

    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    ck, nc, tc = configure("train-gan")
    tc.update(dis_sub_iter=2)
    anet = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
    rt.load_state_dict(P)
    tr = adv.Trainer(anet, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc,
                     mr_source=VolumeSource(val, B, 1234), ct_source=VolumeSource(train, B, 4321),
                     mr_val_source=VolumeSource(val, B, 2234), ct_val_source=VolumeSource(train, B, 5321),
                     test_label_list=lab, test_nii_list=nii)
    tr.train(str(tmp_path / "gan"), restore=False, training_iters=3, epochs=1, display_step=1, dropout=0.75)
    mr, _ = VolumeSource(val, B, 11).next()
    ct, _ = VolumeSource(train, B, 12).next()
    d = tr.loss_value(tr.d_step(mr, ct, 0.75))
    g = tr.loss_value(tr.g_step(ct, 0.75))
    assert np.isfinite(d) and np.isfinite(g), (d, g)
    os.makedirs(str(tmp_path / "gan_test"))
    tr.test_eval(str(tmp_path / "gan_test"), surface_metrics=True)
    assert len(tr.sample_surface_list) == 1
