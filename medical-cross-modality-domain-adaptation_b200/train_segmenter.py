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
    ap.add_argument("--image-summaries", action="store_true",
                    help="also write the reference's TensorBoard image summaries (prediction, input slice, ground truth) every display step")
    a = ap.parse_args(argv)
    logging.basicConfig(level=logging.INFO)
    parallel.init_from_env()
    if a.conv_backend:
        rt.set_conv_backend(a.conv_backend)
    net = drn.Full_DRN(channels=3, n_class=num_cls, batch_size=a.batch_size, cost_kwargs=dict(cost_kwargs))
    print("Network has been built ...")
    train_list, val_list = resolve_lists(a.train_list, a.val_list, a.synthetic)
    trainer = drn.Trainer(net, train_list=train_list, val_list=val_list, num_cls=num_cls, batch_size=a.batch_size, opt_kwargs=dict(opt_kwargs),
                          checkpoint_space=checkpoint_space, optimizer=optimizer, lr_update_flag=False)
    print("Now start training...")
    return trainer.train(output_path=a.output_path, restored_path=a.output_path, training_iters=a.training_iters,
                         epochs=a.epochs, restore=restore, dropout=a.keep_prob, image_summaries=a.image_summaries)


if __name__ == "__main__":
    main()
