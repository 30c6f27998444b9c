"""Why does the held-out hard-Dice gate (tests/test_trajectory_gpu.py) move by more than 1e-3 on some trained models?

Trains the segmenter on the GPU the way the gate does, then looks at the held-out logits of the CUDA path and of the CPU oracle:
magnitude of the logits, distribution of the top-2 margin, distribution of the per-pixel deviation, and which pixels re-label.
Usage (GPU box):  python tests/diag_dice_gate.py --scale 0.25 --rounds 8 --decay 0.7
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=0.25)
    ap.add_argument("--contrast", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--decay", type=float, default=1.0)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--settle", type=int, default=30)
    ap.add_argument("--check", type=int, default=4)
    a = ap.parse_args()
    from tests.models import seg_pair
    from pnp_b200 import runtime as rt
    from pnp_b200.data import SyntheticSource
    from oracle.pnp_graphs import OracleSegmenter
    B = 8
    net, trainer, _, P = seg_pair("auto", B)
    train_src = SyntheticSource(B, seed=1234, num_cls=5, pool=4, contrast=a.contrast, scale=a.scale)
    held = SyntheticSource(B, seed=7777, num_cls=5, pool=8, contrast=a.contrast, scale=a.scale)
    held_dev = [trainer.feed(*held.pool[i]) for i in range(8)]

    from oracle import tf14_torch as T
    from oracle.tf14_numpy import label_decomp

    def exposure(err_scale):
        worst, dices, mx = 0.0, [], 0.0
        with torch.no_grad():
            for xg, yg in held_dev:
                lg = net.forward(xg, 1.0, False, False)
                top = lg.topk(2, dim=3)
                mag = lg.abs().amax(3).clamp_min(1e-12)
                p_flip = torch.exp(-(top.values[..., 0] - top.values[..., 1]) / (err_scale * mag))
                lab = yg.argmax(3)
                for c in range(5):
                    e_c = float((p_flip * ((top.indices[..., 0] == c) | (top.indices[..., 1] == c))).sum())
                    den = int((top.indices[..., 0] == c).sum()) + int((lab == c).sum())
                    worst = max(worst, 2.0 * e_c / max(den, 1))
                dices.append(float(net.dice_eval(lg, yg)[0]))
                mx = max(mx, float(lg.abs().max()))
        return worst, float(np.mean(dices)), mx

    def actual(nb):
        """worst per-class / per-batch |dDice| and re-labelled pixels against the CPU oracle on the first nb held-out batches"""
        orc = OracleSegmenter(rt.state_dict(), B)
        worst, flips = 0.0, 0
        for i in range(nb):
            xs, ys = held.pool[i]
            xg, yg = held_dev[i]
            with torch.no_grad():
                lg = net.forward(xg, 1.0, False, False)
                lo = orc.forward(xs.clone(), 1.0, False)["logits"]
                d_o, arr_o = T.dice_eval(lo.argmax(3), torch.from_numpy(label_decomp(5, ys.numpy())), 5)
                d_g, arr_g = net.dice_eval(lg, yg)
            flips += int((lg.argmax(3).cpu() != lo.argmax(3)).sum())
            worst = max(worst, abs(float(d_g) - float(d_o)), max(abs(float(a_) - float(b_)) for a_, b_ in zip(arr_g, arr_o)))
        return worst, flips

    lr = a.lr
    for r in range(a.rounds):
        trainer.optimizer.set_lr(lr)
        for _ in range(30):
            wce, dice = trainer.train_step(*trainer.feed(*train_src.next()), keep_prob=1.0)
        trainer.optimizer.set_lr(0.0)
        for _ in range(a.settle):
            trainer.train_step(*trainer.feed(*train_src.next()), keep_prob=1.0)
        e5, dv, mx = exposure(1e-5)
        e4 = exposure(1e-4)[0]
        e3 = exposure(3e-5)[0]
        wd, fl = actual(a.check)
        print("round %2d lr %.1e: wce %.4f dice-loss %.4f held-out Dice %.4f max|logit| %.1f | exposure 1e-5: %.2e 3e-5: %.2e 1e-4: %.2e | actual worst dDice %.2e flips %d (%d batches)"
              % (r, lr, float(wce), float(dice), dv, mx, e5, e3, e4, wd, fl, a.check), flush=True)
        lr *= a.decay

    oracle = OracleSegmenter(rt.state_dict(), B)
    xs, ys = held.pool[0]
    xg, yg = held_dev[0]
    with torch.no_grad():
        lg = net.forward(xg, 1.0, False, False).cpu()
        lo = oracle.forward(xs.clone(), 1.0, False)["logits"]
    err = (lg - lo).abs().amax(3)
    top = lo.topk(2, dim=3)
    margin = top.values[..., 0] - top.values[..., 1]
    q = [0.001, 0.01, 0.1, 0.5, 0.9, 0.99, 0.999, 1.0]
    print("max|logit| %.3f ; |top-1 logit| median %.3f" % (float(lo.abs().max()), float(top.values[..., 0].abs().median())))
    print("top-2 margin quantiles  ", " ".join("%g:%.3e" % (p, float(margin.flatten().quantile(p))) for p in q))
    print("per-pixel |dlogit| quant", " ".join("%g:%.3e" % (p, float(err.flatten().quantile(p))) for p in q))
    flip = lg.argmax(3) != lo.argmax(3)
    print("re-labelled pixels: %d of %d ; their margins (max %.3e median %.3e) ; their |dlogit| (max %.3e median %.3e)"
          % (int(flip.sum()), flip.numel(), float(margin[flip].max()) if flip.any() else 0, float(margin[flip].median()) if flip.any() else 0,
             float(err[flip].max()) if flip.any() else 0, float(err[flip].median()) if flip.any() else 0))
    pairs = {}
    for o, m in zip(lo.argmax(3)[flip].tolist(), lg.argmax(3)[flip].tolist()):
        pairs[(o, m)] = pairs.get((o, m), 0) + 1
    print("oracle class -> our class:", pairs)
    for thr in (1e-5, 1e-4, 1e-3, 1e-2, 1e-1):
        print("  pixels with margin < %.0e: %d" % (thr, int((margin < thr).sum())))
    zero = (lo.abs().amax(3) < 1e-6)
    print("pixels whose oracle logits are all ~0: %d ; exact ties in the oracle: %d" % (int(zero.sum()), int((margin == 0).sum())))
    # where the error comes from: relative deviation of the logits per pixel against that pixel's own magnitude
    rel = err / lo.abs().amax(3).clamp_min(1e-12)
    print("per-pixel |dlogit| / max_c|logit| quantiles", " ".join("%g:%.3e" % (p, float(rel.flatten().quantile(p))) for p in q))


if __name__ == "__main__":
    main()
