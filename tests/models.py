"""The model-level builders of the parity tests: the product's segmenter / adversarial network and trainer next to the CPU
oracle on identical seeded initial variables, and the loss and variable comparisons between them."""
import numpy as np
import torch

from tests.util import rel_err


def bn_noise(P, bns, seed):
    rng = np.random.RandomState(seed)
    for n, c in bns:   # non-trivial BN state so that inference-mode BN is really exercised
        P[n + "/gamma"] = (1 + 0.2 * rng.randn(c)).astype(np.float32)
        P[n + "/beta"] = (0.1 * rng.randn(c)).astype(np.float32)
        P[n + "/moving_mean"] = (0.05 * rng.randn(c)).astype(np.float32)
        P[n + "/moving_variance"] = (1 + 0.2 * rng.rand(c)).astype(np.float32)


def adv_pair(backend, lam, phase, B, with_oracle=True, lr=3e-4, dis_sub_iter=1, o64=False):
    """-> (net, trainer, oracle); o64: the oracle carries an fp64 companion as oracle.o64"""
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import OracleAdversarial, init_numpy_params
    rt.set_conv_backend(backend)
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    for n, s in ws:   # keep the critic weights inside the clip range so the clip is exercised but not dominant
        if "cls" in n:
            P[n] = np.clip(P[n] * 0.5, -0.05, 0.05).astype(np.float32)
    ck, nc, tc = configure(phase)
    ck["lambda_mask_loss"] = lam
    tc["dis_sub_iter"] = dis_sub_iter
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc, critic_keep_prob=1.0)
    rt.load_state_dict(P)
    trainer = adv.Trainer(net, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": lr}, train_config=tc)
    oracle = None
    if with_oracle:
        kw = dict(lambda_mask_loss=lam, dis_sub_iter=dis_sub_iter, gen_sub_iter=1, critic_keep_prob=1.0, lr=lr)
        oracle = OracleAdversarial(P, B, **kw)
        if o64:
            oracle.o64 = OracleAdversarial(P, B, dtype=torch.float64, **kw)
    return net, trainer, oracle


def seg_pair(backend, B, lr=1e-3, dtype=torch.float32):
    """-> (net, trainer, oracle, initial variables); dtype: the oracle's"""
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, source_segmenter as seg
    from oracle.pnp_graphs import OracleSegmenter, init_numpy_params
    rt.set_conv_backend(backend)
    ws, bns = OracleSegmenter.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 5)
    ck = {"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0, "regularizer": 1e-4}
    net = seg.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=dict(ck))
    rt.load_state_dict(P)
    trainer = seg.Trainer(net, [], [], num_cls=5, batch_size=B, optimizer="adam", opt_kwargs={"learning_rate": lr})
    return net, trainer, OracleSegmenter(P, B, dtype=dtype, lr=lr), P


def loss_close(name, got, ref, scale_floor, tol=1e-3):
    den = max(abs(ref), scale_floor)
    e = abs(got - ref) / den
    print("  %-34s %.6e (oracle %.6e)  err/scale %.2e (tol %.0e)" % (name, got, ref, e, tol))
    assert np.isfinite(got) and e <= tol, (name, got, ref, e)
    return e


def state_close(rt, oracle, tol, only=None, norm=rel_err, label="worst variable: {name} err {err:.3e} (tol {tol:.0e})"):
    """the largest error `norm` of a product variable against the oracle's, printed with `label`"""
    ref, got = oracle.ps.to_numpy(), rt.state_dict()
    worst, wname = 0.0, None
    for n in ref:
        if only and not only(n):
            continue
        e = norm(torch.tensor(got[n]), torch.tensor(ref[n]))
        if e > worst:
            worst, wname = e, n
    print("  " + label.format(name=wname, err=worst, tol=tol))
    assert worst <= tol, (wname, worst)
    return worst
