"""Cost of the weights' moving average (Trainer(ema_decay=...), elementwise.cu pnp_ema_advance / pnp_ema_update) on the card it
runs on, in one run:
* `pnp_ema_update` alone at the segmenter's coverage (its Adam arena plus every batch-norm moving statistic) and at the GAN's (the
  G arena plus the DAM's statistics), as time per launch and GB/s at 12 bytes per covered float (read shadow, read live, write
  shadow) against the H100 SXM data-sheet 3.35 TB/s;
* the captured segmenter Adam step at B = 16 and the captured joint D + G step at B = 8 (config 2 and 4 of bench.py), each captured
  with the average on and off on the same trainer, replayed in alternating rounds.
Times are CUDA events, medians over `--reps` rounds.  Prints the card name and its power limit with the numbers, one JSON line at
the end.

    python scripts/bench_ema.py [--launches 200] [--steps 20] [--reps 9]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

HBM_TBS = 3.35


def _events(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n                    # ms per call


def _update_cost(ema, launches, reps):
    from pnp_b200 import runtime as rt
    from pnp_b200._C import call, ptr

    def once():
        call("pnp_ema_update", ptr(ema.shadow), ptr(ema.arena.theta), ema.arena.total, ptr(ema.table), ema.table_n, ptr(ema.c),
             rt.stream())
    once()
    ms = statistics.median(_events(once, launches) for _ in range(reps))
    floats = ema.arena.total + sum(v.numel() for v in ema.extra)
    return {"arena_floats": ema.arena.total, "stat_floats": sum(v.numel() for v in ema.extra), "stat_chunks": ema.table_n,
            "update_ms": ms, "GBps": 12.0 * floats / (ms * 1e-3) / 1e9, "share_of_3.35TBps": 12.0 * floats / (ms * 1e-3) / (HBM_TBS * 1e12)}


def _step_cost(replay_on, replay_off, steps, reps):
    on, off = [], []
    for _ in range(reps):
        on.append(_events(replay_on, steps))
        off.append(_events(replay_off, steps))
    m_on, m_off = statistics.median(on), statistics.median(off)
    return {"step_ms_ema_on": m_on, "step_ms_ema_off": m_off, "overhead_pct": 100.0 * (m_on - m_off) / m_off}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark measures the GPU and needs one"
    import pnp_b200  # noqa: F401
    from pnp_b200 import adversarial as adv, runtime as rt, source_segmenter as seg
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import synthetic_images, synthetic_labels
    from bench_volume_source import _power_limit
    card, power = torch.cuda.get_device_name(0), _power_limit()
    print("card: %s, power limit %s" % (card, power))
    res = {"card": card, "power_limit": power}
    rt.set_conv_backend("auto")
    rt.manual_seed(1)

    # segmenter, config 2: Adam step at B = 16
    B = 16
    net = seg.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs={"cross_flag": True, "miu_cross": 1.0, "dice_flag": True,
                                                                          "miu_dice": 1.0, "regularizer": 1e-4})
    tr = seg.Trainer(net, [], [], num_cls=5, batch_size=B, optimizer="adam", opt_kwargs={"learning_rate": 1e-3}, ema_decay=0.999)
    res["segmenter_update"] = _update_cost(tr.ema, a.launches, a.reps)
    print("segmenter pnp_ema_update: %s" % res["segmenter_update"])
    x = synthetic_images(B, 1234).cuda()
    y = torch.nn.functional.one_hot(torch.from_numpy(synthetic_labels(B, 99)), 5).float().cuda()
    ema = tr.ema
    assert tr.capture_train_step(x, y, 0.75)
    g_on = tr._graph
    tr.ema = None
    assert tr.capture_train_step(x, y, 0.75)
    g_off = tr._graph
    tr.ema = ema
    res["segmenter_step_B16"] = _step_cost(lambda: g_on.replay(x, y), lambda: g_off.replay(x, y), a.steps, a.reps)
    print("segmenter captured Adam step: %s" % res["segmenter_step_B16"])
    del tr, net, g_on, g_off, ema
    torch.cuda.empty_cache()

    # GAN, config 4: joint D + G step at B = 8
    B = 8
    ck, nc, tc = configure("train-gan")
    tc["dis_sub_iter"] = 1
    anet = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc, stddev=0.05, stddev_plain=0.05)
    atr = adv.Trainer(anet, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc, ema_decay=0.999)
    res["gan_update"] = _update_cost(atr.ema, a.launches, a.reps)
    print("GAN pnp_ema_update: %s" % res["gan_update"])
    mr, ct, ct2 = synthetic_images(B, 1234).cuda(), synthetic_images(B, 4321, 0.3, 0.8).cuda(), synthetic_images(B, 4322, 0.3, 0.8).cuda()
    ema = atr.ema
    assert atr.capture_joint_step(mr, ct, 0.75)
    g_on = atr._graph
    atr.ema = None
    assert atr.capture_joint_step(mr, ct, 0.75)
    g_off = atr._graph
    atr.ema = ema
    res["gan_joint_step_B8"] = _step_cost(lambda: g_on.replay(mr, ct, ct2), lambda: g_off.replay(mr, ct, ct2), a.steps, a.reps)
    print("GAN captured joint step: %s" % res["gan_joint_step_B8"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
