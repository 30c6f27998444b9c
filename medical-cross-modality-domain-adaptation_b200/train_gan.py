"""Entry point mirroring the reference's train_gan.py (:24-157): `--phase pre-train | train-gan | fine-tune`
with the reference's configuration dictionaries and per-phase overrides (keys kept verbatim)."""
import argparse
import os
import logging

from . import adversarial as drn
from . import parallel
from . import runtime as rt

rate = 0.3
date = "1221"

cost_kwargs = {
    "regularizer": 1e-4,        # L2 regulariser of the (frozen) segmentation model -- monitoring only
    "gan_regularizer": 1e-4,    # L2 regulariser of the WGAN variables
    "miu_gen": 0.002,
    "miu_dis": 0.002,
    "lambda_mask_loss": None,   # trade-off of the mask critic, set per phase
}
opt_kwargs = {"learning_rate": 3e-4}
network_config = {
    "mr_front_trainable": False, "joint_trainable": False, "ct_front_trainable": None,
    "cls_trainable": True, "m_cls_trainable": True, "restore_skip_kwd": ["Adam", "RMS", "cls"],
}
train_config = {
    "restore_from_baseline": None, "copy_main": None, "clear_rms": None, "lr_update": None,
    "dis_interval": 1, "gen_interval": 1, "dis_sub_iter": 20, "gen_sub_iter": 1,
    "tag": "gan-" + str(rate) + "_" + date, "iter_upd_interval": 300, "dis_sub_iter_inc": 1, "gen_sub_iter_inc": 0,
    "lr_decay_factor": 0.98, "checkpoint_space": 100, "training_iters": 200, "epochs": 600,
}


def configure(phase):
    """train_gan.py:85-129 -- returns fresh (cost_kwargs, network_config, train_config) for a phase"""
    ck, nc, tc = dict(cost_kwargs), dict(network_config), dict(train_config)
    if phase == 'pre-train':
        nc["ct_front_trainable"] = False
        tc.update(restore_from_baseline=True, copy_main=True, clear_rms=True, lr_update=True, gen_interval=0, dis_sub_iter=1,
                  dis_sub_iter_inc=0, checkpoint_space=2000, training_iters=201, epochs=100)
        ck["lambda_mask_loss"] = 0
    elif phase == 'train-gan':
        nc["ct_front_trainable"] = True
        tc.update(restore_from_baseline=False, copy_main=False, clear_rms=False, lr_update=True, tag=tc["tag"] + "-gan")
        ck["lambda_mask_loss"] = rate
    elif phase == 'fine-tune':
        nc["ct_front_trainable"] = True
        # the reference writes `training_config["lr_update"]` here (NameError, train_gan.py:121); intent restored
        tc.update(restore_from_baseline=False, copy_main=False, clear_rms=False, lr_update=False, gen_interval=1, dis_sub_iter=30,
                  tag=tc["tag"] + "-fine_tune")
        ck["lambda_mask_loss"] = rate
    else:
        raise Exception("Please set a training phase!")
    return ck, nc, tc


def main(phase, argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--phase", type=str, default=phase)
    ap.add_argument("--batch-size", type=int, default=6)
    ap.add_argument("--training-iters", type=int, default=None)
    ap.add_argument("--epochs", type=int, default=None)
    ap.add_argument("--keep-prob", type=float, default=0.75)
    ap.add_argument("--conv-backend", default=None, choices=["auto", "simt", "tc3", "tc1"])
    ap.add_argument("--lists", default="./lists", help="directory of mr_train_list, mr_val_list, ct_train_list, ct_val_list")
    ap.add_argument("--synthetic", action="store_true", help="ignore the list files and train on the synthetic sources")
    ap.add_argument("--volumes", action="store_true",
                    help="draw freshly augmented slices on the GPU from the NIfTI pairs of <lists>/{mr,ct}_{train,val}_volumes")
    ap.add_argument("--elastic", action="store_true",
                    help="with --volumes: add smooth random elastic deformations to the MR and CT training slices (preprocess.py)")
    ap.add_argument("--intensity", action="store_true",
                    help="with --volumes: add a smooth bias field, a contrast and an offset to the MR and CT training slices")
    ap.add_argument("--image-summaries", action="store_true",
                    help="also write the reference's TensorBoard image summaries (prediction, input slice, ground truth) every display step")
    ap.add_argument("--ema-decay", type=float, default=None, metavar="D",
                    help="keep an exponential moving average of the trained weights with this decay (0 < D < 1): checkpointed, "
                         "monitored as ema_* scalars and written as averaged-weights checkpoints *_ema.npz")
    a = ap.parse_args(argv)
    if (a.elastic or a.intensity) and not a.volumes:
        ap.error("--elastic / --intensity augment the slices drawn with --volumes; give --volumes")
    if a.ema_decay is not None:
        if a.phase == "pre-train":
            ap.error("--ema-decay averages the generator's weights; the pre-train phase runs no generator step")
        if not 0.0 < a.ema_decay < 1.0:
            ap.error("--ema-decay must lie in (0, 1)")
    logging.basicConfig(level=logging.INFO)
    parallel.init_from_env()
    if a.conv_backend:
        rt.set_conv_backend(a.conv_backend)
    ck, nc, tc = configure(a.phase)
    num_cls = 5
    out = "./tmp_exps/mr2ct" + date + str(rate)[0] + str(rate)[2]
    net = drn.Full_DRN(channels=3, batch_size=a.batch_size, n_class=num_cls, cost_kwargs=ck, network_config=nc)
    print("Network has been built ...")
    # train_gan.py:69-72; the four variable-name lists the reference also reads (:74-77) are not inputs here: the MR -> CT copy
    # pairs and the BN hand-over pairs are derived from the graph (and pinned to those very lists by tests/test_reference_graph_trace.py)
    from .train_segmenter import resolve_lists
    mr_train, mr_val, ct_train, ct_val = resolve_lists(*[os.path.join(a.lists, n) for n in
                                                         ("mr_train_list", "mr_val_list", "ct_train_list", "ct_val_list")], a.synthetic)
    sources = {}
    if a.volumes:
        # each stream keeps the seed of the stream it replaces (adversarial.Trainer.train: 1234 / 4321 / 2234 / 5321 + rank)
        from .train_segmenter import volume_source
        rank = parallel.DataParallel().rank
        # the opt-in augmentations apply to the two training streams only
        aug = {"elastic": a.elastic, "intensity": a.intensity}
        for key, name, seed, kw in (("mr_source", "mr_train_volumes", 1234, aug), ("ct_source", "ct_train_volumes", 4321, aug),
                                    ("mr_val_source", "mr_val_volumes", 2234, {}), ("ct_val_source", "ct_val_volumes", 5321, {})):
            sources[key] = volume_source(os.path.join(a.lists, name), a.batch_size, seed + rank, **kw)
    trainer = drn.Trainer(net, mr_train, mr_val, ct_train, ct_val, num_cls=num_cls, batch_size=a.batch_size,
                          opt_kwargs=dict(opt_kwargs), train_config=tc, ema_decay=a.ema_decay, **sources)
    print("Now start training...")
    return trainer.train(output_path=out, restored_path=out, training_iters=a.training_iters or tc["training_iters"],
                         epochs=a.epochs or tc["epochs"], dropout=a.keep_prob, image_summaries=a.image_summaries)
