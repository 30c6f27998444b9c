"""Entry point mirroring the reference's train_segmenter.py (:22-79): source-only (MR) segmenter training
with the same configuration literals.  `python train_segmenter.py [--batch-size N] ...`
Like the reference it reads ./lists/mr_train_list and ./lists/mr_val_list (text files of single-example TFRecord paths,
README.md:49-64) when they exist; without them -- or with --synthetic -- the synthetic source stands in.
The reference's `os.system('tensorboard ...')` side effect (:69-70) is intentionally dropped; the scalar summaries are written
as event files under <output_path>/train_log and val_log."""
import argparse
import logging
import os

from . import parallel
from .lib import _read_lists
from . import runtime as rt
from . import source_segmenter as drn

train_fid = "./lists/mr_train_list"
val_fid = "./lists/mr_val_list"
output_path = "./tmp_exps/mr_baseline"
restore = True  # the reference restores even on a first run and falls through to "start from beginning" (:28,73)
num_cls = 5
batch_size = 10
training_iters = 10            # train_segmenter.py:33
epochs = 5000
checkpoint_space = 1500
optimizer = 'adam'
cost_kwargs = {"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0, "regularizer": 1e-4}
opt_kwargs = {"learning_rate": 1e-3}


def resolve_lists(*fids_and_flag):
    """_read_lists on each list file (train_segmenter.py:60-61, train_gan.py:69-72).  A missing list file means "no data here": the
    synthetic source is used.  A list whose first entry does not exist is an error -- silently training on synthetic data while
    the user believes the dataset is being read would be worse than stopping."""
    *fids, synthetic = fids_and_flag
    out = []
    for fid in fids:
        lst = None if synthetic else _read_lists(fid)
        if lst:
            if not os.path.isfile(lst[0]):
                raise IOError("%s lists %s, which does not exist (pass --synthetic to train without the dataset)" % (fid, lst[0]))
            logging.info("%s: %d TFRecord files" % (fid, len(lst)))
        out.append(lst or [])
    return out


def volume_source(pairs_file, batch_size, seed, elastic=False, intensity=False):
    """data.VolumeSource over the `image label` pairs of a list file (elastic / intensity: its opt-in augmentations)"""
    from .data import VolumeSource
    from .preprocess import read_pairs
    pairs = read_pairs(pairs_file)
    logging.info("%s: %d volume pairs" % (pairs_file, len(pairs)))
    return VolumeSource(pairs, batch_size, seed, elastic=elastic, intensity=intensity)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=batch_size)
    ap.add_argument("--training-iters", type=int, default=training_iters)
    ap.add_argument("--epochs", type=int, default=epochs)
    ap.add_argument("--keep-prob", type=float, default=0.75)
    ap.add_argument("--conv-backend", default=None, choices=["auto", "simt", "tc3", "tc1"])
    ap.add_argument("--output-path", default=output_path)
    ap.add_argument("--train-list", default=train_fid)
    ap.add_argument("--val-list", default=val_fid)
    ap.add_argument("--synthetic", action="store_true", help="ignore the list files and train on the synthetic source")
    ap.add_argument("--train-volumes", default=None,
                    help="file of `image label` NIfTI pairs: draw freshly augmented training slices from these volumes on the GPU")
    ap.add_argument("--val-volumes", default=None, help="file of `image label` NIfTI pairs: validation slices from these volumes")
    ap.add_argument("--elastic", action="store_true",
                    help="with --train-volumes: add smooth random elastic deformations to the training slices (preprocess.py)")
    ap.add_argument("--intensity", action="store_true",
                    help="with --train-volumes: add a smooth bias field, a contrast and an offset to the training slices")
    ap.add_argument("--image-summaries", action="store_true",
                    help="also write the reference's TensorBoard image summaries (prediction, input slice, ground truth) every display step")
    ap.add_argument("--ema-decay", type=float, default=None, metavar="D",
                    help="keep an exponential moving average of the trained weights with this decay (0 < D < 1): checkpointed, "
                         "monitored as ema_* scalars and written as averaged-weights checkpoints *_ema.npz")
    a = ap.parse_args(argv)
    if (a.elastic or a.intensity) and not a.train_volumes:
        ap.error("--elastic / --intensity augment the slices drawn from --train-volumes; give --train-volumes")
    if a.ema_decay is not None and not 0.0 < a.ema_decay < 1.0:
        ap.error("--ema-decay must lie in (0, 1)")
    logging.basicConfig(level=logging.INFO)
    parallel.init_from_env()
    if a.conv_backend:
        rt.set_conv_backend(a.conv_backend)
    net = drn.Full_DRN(channels=3, n_class=num_cls, batch_size=a.batch_size, cost_kwargs=dict(cost_kwargs))
    print("Network has been built ...")
    train_list, val_list = resolve_lists(a.train_list, a.val_list, a.synthetic)
    # VolumeSource streams take the seeds of the streams they replace (source_segmenter.Trainer.train: 1234 / 4321 + rank)
    # the opt-in augmentations apply to the training stream only
    rank = parallel.DataParallel().rank
    sources = {k: volume_source(path, a.batch_size, seed + rank, **aug) for k, path, seed, aug in
               (("source", a.train_volumes, 1234, {"elastic": a.elastic, "intensity": a.intensity}),
                ("val_source", a.val_volumes, 4321, {})) if path}
    trainer = drn.Trainer(net, train_list=train_list, val_list=val_list, num_cls=num_cls, batch_size=a.batch_size, opt_kwargs=dict(opt_kwargs),
                          checkpoint_space=checkpoint_space, optimizer=optimizer, lr_update_flag=False, ema_decay=a.ema_decay,
                          **sources)
    print("Now start training...")
    return trainer.train(output_path=a.output_path, restored_path=a.output_path, training_iters=a.training_iters,
                         epochs=a.epochs, restore=restore, dropout=a.keep_prob, image_summaries=a.image_summaries)


if __name__ == "__main__":
    main()
