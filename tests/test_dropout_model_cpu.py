"""CPU side of tests/test_dropout_model_gpu.py: the mask stand-in (tests/models.PhiloxMasks) and the order in which it hands out
stream ids.

  * site census: the (output shape, keep) sequence the stand-in sees while the oracle runs a segment (each stream), the feature
    critic and the mask critic equals, in order, the convolutions with keep != 1 that the reference's own graph creates
    (tests/golden/reference_graph_trace.json, recorded by executing the reference's graph code).  So the stream ids the oracle
    assigns follow the reference's layer order, not the product's.  The sub-graphs run on meta tensors; the whole steps run at
    B = 1 and must draw the site counts the GPU tests derive their ids from.
  * stand-in semantics: the mask is dropout_mult's, i.e. T.dropout(x, keep, mask=kept) up to the rounding of 1/keep to fp32, and
    the fp32 and fp64 oracles of one step share the cached mask.
"""
import json
import os

import numpy as np
import pytest
import torch

from tests.models import PhiloxMasks
from tests.test_dropout_model_gpu import CLS, KEEP, MASK, N_D, N_G, SEG

HERE = os.path.dirname(os.path.abspath(__file__))


def _ref_sites(section):
    """[(out [H, W, C], keep)] of the reference's convolutions with keep != 1 in one trace section; the keep_prob placeholder
    stands for the keep the test feeds"""
    with open(os.path.join(HERE, "golden", "reference_graph_trace.json")) as f:
        ev = json.load(f)["events"]
    out = []
    for e in ev:
        if e["section"] == section and e["op"] == "conv":
            keep = KEEP if e["keep"] == "ph:keep_prob" else float(e["keep"])
            if keep != 1.0:
                out.append((list(e["out"]), keep))
    return out


def _sites(seen):
    return [(list(s[1:]), k) for s, k in seen if k != 1.0]


def _meta_oracle(B):
    """an adversarial oracle (critic keep 0.75) whose variables live on the meta device: shapes only"""
    from oracle.pnp_graphs import OracleAdversarial
    o = OracleAdversarial({}, B, lambda_mask_loss=0.3, critic_keep_prob=0.75)
    o.ps.w = {k: v.detach().to("meta") for k, v in o.ps.w.items()}
    for bn in o.ps.bn.values():
        bn.gamma, bn.beta = bn.gamma.detach().to("meta"), bn.beta.detach().to("meta")
        bn.moving_mean, bn.moving_var = bn.moving_mean.to("meta"), bn.moving_var.to("meta")
    return o


@pytest.fixture
def masks(monkeypatch):
    from oracle import tf14_torch as T
    m = PhiloxMasks(12345)
    monkeypatch.setattr(T, "dropout", m)
    return m.at(1, 0)


def test_site_census_matches_the_reference_graph(masks):
    """zip_network#1 holds both fronts (MR then CT, 21 sites each); second_half#1 is the CT stream's call, #2 the MR stream's
    (11 sites and the keep-1 output convolution); create_classifier#* 16 sites, create_mask_critic#* 8"""
    o = _meta_oracle(1)
    x = torch.empty(1, 256, 256, 3, device="meta")
    zipn = _ref_sites("create_zip_network#1")
    assert len(zipn) == 2 * 21
    want = {"mr": zipn[:21] + _ref_sites("create_second_half#2"), "ct": zipn[21:] + _ref_sites("create_second_half#1")}
    with torch.no_grad():
        for stream in ("mr", "ct"):
            masks.seen = []
            f = o.segment(x, stream, KEEP, False)
            assert _sites(masks.seen) == want[stream], stream
            assert masks.seen[-1] == ((1, 256, 256, 5), 1.0)           # the output convolution: keep 1, no stream id
            assert len(want[stream]) == SEG
        masks.seen = []
        o.classifier(f["c4_2"], f["c6_2"], f["b7"], f["c9_2"], f["logits"])
        assert _sites(masks.seen) == _ref_sites("create_classifier#1") == _ref_sites("create_classifier#2")
        assert len(masks.seen) == CLS
        masks.seen = []
        o.mask_critic(f["logits"])
        assert _sites(masks.seen) == _ref_sites("create_mask_critic#1") == _ref_sites("create_mask_critic#2")
        assert len(masks.seen) == MASK
    assert masks.sid == 2 * SEG + CLS + MASK


def test_step_site_counts(masks):
    """the whole oracle steps (B = 1): every site draws one id, in the order the reference's sub-graphs run in each step"""
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter, init_numpy_params, synthetic_images, synthetic_labels
    from oracle.tf14_numpy import label_decomp
    mr, ct = synthetic_images(1, 1), synthetic_images(1, 2)
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    zipn = _ref_sites("create_zip_network#1")
    seg_mr, seg_ct = zipn[:21] + _ref_sites("create_second_half#2"), zipn[21:] + _ref_sites("create_second_half#1")
    cls, msk = _ref_sites("create_classifier#1"), _ref_sites("create_mask_critic#1")
    for lam in (0.0, 0.3):
        o = OracleAdversarial(P, 1, lambda_mask_loss=lam, critic_keep_prob=0.75)
        masks.at(1, 0).seen = []
        o.d_step(mr, ct, KEEP)
        assert masks.sid == N_D[lam]
        assert _sites(masks.seen) == seg_mr + seg_ct + cls + cls + (msk + msk if lam else [])
        if lam:
            masks.at(2, 0).seen = []
            o.g_step(ct, KEEP)
            assert masks.sid == N_G
            assert _sites(masks.seen) == seg_ct + cls + msk
    ws, bns = OracleSegmenter.layout()
    o = OracleSegmenter(init_numpy_params(ws, bns, 0, 0.05), 1)
    masks.at(1, 0).seen = []
    o.train_step(synthetic_images(1, 3), torch.from_numpy(label_decomp(5, synthetic_labels(1, 4))), KEEP)
    assert masks.sid == SEG
    assert _sites(masks.seen) == seg_mr              # the segmenter is the MR stream's layer sequence


@pytest.mark.parametrize("keep", [0.5, 0.75, 0.6137])
def test_stand_in_is_the_library_mask(keep):
    from oracle import philox, tf14_torch as T
    m = PhiloxMasks(-7)                                  # manual_seed keeps the low 63 bits
    assert m.s0 == (-7) & (2 ** 63 - 1)
    x = torch.randn(2, 8, 8, 16, generator=torch.Generator().manual_seed(3))
    m.at(3, 5)
    y = m(x, keep)
    assert m.sid == 6
    seed = philox.seed_advance(m.s0, 3)
    kept = philox.draws16(seed, 6, x.numel()) < philox.keep_threshold(keep)
    assert 0 < kept.sum() < x.numel()
    kept = torch.from_numpy(kept.reshape(x.shape))
    ref = T.dropout(x, keep, mask=kept.float())          # x * kept / keep
    assert torch.equal(y == 0, ~kept | (x == 0))
    assert torch.equal(y, x * torch.where(kept, float(philox.inv_keep(keep)), 0.0).float())
    torch.testing.assert_close(y, ref, rtol=2.0 ** -23, atol=0.0)        # 1/keep rounded to fp32 first
    # the fp64 oracle reads the same cached mask and multiplies by the exact fp32 values 0 and fl32(1/keep)
    assert len(m.cache) == 1
    m.at(3, 5)
    y64 = m(x.double(), keep)
    assert len(m.cache) == 1 and y64.dtype == torch.float64
    assert torch.equal(y64, x.double() * torch.where(kept, float(philox.inv_keep(keep)), 0.0).double())
    # keep >= 1 is the identity and draws no id; moving to another step drops the cached masks
    assert m(x, 1.0) is x and m.sid == 6
    m.at(4, 0)
    assert m.cache == {}
