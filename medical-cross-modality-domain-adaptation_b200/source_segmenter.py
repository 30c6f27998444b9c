"""Source-only dilated-residual segmenter and its Adam training step -- the H100-native counterpart of
the reference's source_segmenter.py (Full_DRN :48-301, Trainer :303-675), eager instead of TF-1 graph.

Mapping of the reference's graph attributes (evaluated there through sess.run + feed_dict):
    net.x / net.y / net.keep_prob / net.main_bn / net.adapt_bn  -> arguments of net.forward()/net.losses()
    net.predicter, net.compact_pred, net.cost, net.regularizer_loss, net.weighted_loss, net.dice_loss,
    net.dice_eval[_arr], net.confusion_matrix                   -> methods of the same name
Out of scope (SURVEY 2.1 row 4): TFRecord queues, TensorBoard summaries, NIfTI test_eval (which does not
even parse in the reference, source_segmenter.py:611).
"""
import logging
import os
import time

import numpy as np
import torch

from . import functional as F
from . import layers as L
from . import runtime as rt
from . import optim
from . import parallel
from . import summary
from .data import pick_source, to_device
from .ema import EMA
from .lib import _label_decomp, save_checkpoint
from .networks import FRONT, BACK, SegmenterHalf, SegmenterTail

raw_size = [256, 256, 3]
volume_size = [256, 256, 3]
label_size = [256, 256, 1]


class Full_DRN(object):
    """source_segmenter.py:48-273.  cost_kwargs: dice_flag, cross_flag, miu_dice, miu_cross, regularizer."""

    def __init__(self, channels, n_class, batch_size, adapt_module=True, main_trainable=True, adapt_trainable=True,
                 cost_kwargs={}, **kwargs):
        rt.reset_default_graph()
        self.n_class = n_class
        self.batch_size = batch_size
        self.main_trainable = main_trainable
        self.adapt_trainable = adapt_trainable
        stddev = kwargs.get("stddev", 0.01)                     # layers.py:47
        counter = [0]

        def anon(gi, blk, kind):
            # tf.contrib.layers.batch_norm(scope=None): top-level BatchNorm, BatchNorm_1, ... in creation order
            def one():
                k = counter[0]
                counter[0] += 1
                return "/BatchNorm" if k == 0 else "/BatchNorm_%d" % k
            return one() if kind == "b" else (one(), one())

        # groups 1-4 use adapt_trainable, 5+ main_trainable (source_segmenter.py:91-161)
        self.front_a = SegmenterHalf({g: FRONT[g] for g in (1, 2, 3, 4)}, "group_%d", channels, anon, adapt_trainable, stddev)
        self.front_b = SegmenterHalf({g: FRONT[g] for g in (5, 6)}, "group_%d", self.front_a.out_channels, anon, main_trainable, stddev)
        self.back = SegmenterHalf(BACK, "group_%d", self.front_b.out_channels, anon, main_trainable, stddev)
        self.tail = SegmenterTail(n_class, main_trainable, stddev)
        ws = self.front_a.weights + self.front_b.weights + self.back.weights + self.tail.weights
        # conv_weights with the reference's quirk (source_segmenter.py:132-135): wr4_4 twice, wr4_3 never
        wr4_3 = rt.graph.vars["group_4/Variable_2"]
        wr4_4 = rt.graph.vars["group_4/Variable_3"]
        self.conv_weights = []
        for w in ws:
            if w is wr4_3:
                continue
            self.conv_weights.append(w)
            if w is wr4_4:
                self.conv_weights.append(w)
        self.all_weights = ws

        ck = dict(cost_kwargs)
        self.dice_flag = ck.pop("dice_flag", True)
        self.cross_flag = ck.pop("cross_flag", False)
        self.miu_dice = ck.pop("miu_dice", None)
        self.miu_cross = ck.pop("miu_cross", None)
        self.reg_coeff = ck.pop("regularizer", 1e-4)

    # ---- graph ---------------------------------------------------------------------------------------
    def forward(self, x, keep_prob=1.0, main_bn=True, adapt_bn=True, return_taps=False):
        """create_network (source_segmenter.py:88-209) -> logits [B,256,256,n_class]"""
        h, t1 = self.front_a.run(x, keep_prob, adapt_bn, self.adapt_trainable)
        h, t2 = self.front_b.run(h, keep_prob, main_bn, self.main_trainable)
        h, t3 = self.back.run(h, keep_prob, main_bn, self.main_trainable)
        logits = self.tail.run(h, keep_prob, self.batch_size)
        if return_taps:
            return logits, {"c4_2": t1[4], "c6_2": t2[6], "b7": t3[7], "b8": t3[8], "c9_2": t3[9]}
        return logits

    __call__ = forward

    def predicter(self, logits):
        return L.pixel_wise_softmax_2(logits)

    def compact_pred(self, logits):
        return torch.argmax(self.predicter(logits), 3)

    def losses(self, logits, y):
        """(cost, weighted_loss, dice_loss) -- source_segmenter.py:211-273"""
        wce, dice = F.seg_losses(logits, y)
        # values only: a reference to the tensors themselves would keep the step's autograd graph alive, and with it the
        # variables' gradient accumulators, which remember the stream they were created on.  A CUDA-graph capture that follows
        # a step on another stream would then end its backward pass by waiting on that stream, which invalidates the capture
        self.weighted_loss, self.dice_loss = wce.detach(), dice.detach()
        return wce, dice

    def cost_value(self, wce, dice):
        c = 0.0
        if self.cross_flag is True:
            c = c + self.miu_cross * float(wce)
        if self.dice_flag is True:
            c = c + self.miu_dice * float(dice)
        return c

    def regularizer_loss(self):
        return self.reg_coeff * float(F.l2_loss_sum(self.conv_weights).item())

    def dice_eval(self, logits, y):
        from .lib import _dice_eval
        return _dice_eval(logits, y, self.n_class)

    def confusion_matrix(self, logits, y):
        return F.confusion_counts(logits, y)

    def weight_decay_table(self, variables):
        """per-variable coefficient of the L2 term's gradient: reg_coeff * multiplicity in conv_weights"""
        mult = {}
        for w in self.conv_weights:
            mult[id(w)] = mult.get(id(w), 0) + 1
        return [self.reg_coeff * mult.get(id(v), 0) for v in variables]

    def restore(self, model_path):
        """source_segmenter.py:275-300 with relaxation: load every stored variable whose name we know."""
        d = dict(np.load(model_path))
        self.last_restored = d
        missing = rt.load_state_dict({k: v for k, v in d.items() if k in rt.graph.vars}, strict=False)
        logging.info("Model restored from file: %s (%d unknown names skipped)" % (model_path, len(missing)))


class Trainer(object):
    """source_segmenter.py:303-675, re-hosted: same constructor / train() arguments; inputs come from a
    synthetic source unless `source` is given (anything with .next() -> (images, int labels))."""

    def __init__(self, net, train_list, val_list, num_cls, batch_size, test_nii_list=None, test_label_list=None,
                 optimizer="momentum", opt_kwargs={}, num_epochs=100, checkpoint_space=500, lr_update_flag=False, source=None,
                 val_source=None, ema_decay=None):
        """`ema_decay`: keep an exponential moving average (ema.EMA) of the optimizer's variables and of every batch-norm moving
        statistic, updated after every optimizer step, checkpointed, monitored and written as averaged-weights checkpoints;
        None: no average"""
        self.net = net
        self.batch_size = batch_size
        self.num_cls = num_cls
        self.checkpoint_space = checkpoint_space
        self.opt_kwargs = dict(opt_kwargs)
        self.lr_update_flag = lr_update_flag
        self.train_list, self.val_list = train_list, val_list
        self.test_nii_list, self.test_label_list = test_nii_list, test_label_list
        if optimizer not in ("adam", "momentum"):
            raise ValueError("optimizer must be 'adam' or 'momentum' (source_segmenter.py:359-381)")
        self.optimizer_name = optimizer
        self.source, self.val_source = source, val_source
        self.global_step = 0
        self.dp = parallel.DataParallel()
        self._graph = None           # the captured train step (runtime.StepGraph), None: eager
        self._build_optimizer()
        self.ema = None if ema_decay is None else EMA(
            self.arena, [v for v in rt.global_variables() if v.pnp_kind == "bn_moving"], ema_decay)

    def _build_optimizer(self):
        """source_segmenter.py:357-381: Adam over every trainable variable, loss = cost + regularizer"""
        tv = [v for v in rt.global_variables() if v.pnp_trainable]
        self.trainables = tv
        self.arena = optim.Arena(tv)
        self.dp.attach(self.arena)
        if self.optimizer_name == "momentum":
            # source_segmenter.py:360-372; decay_steps = training_iters is bound when train() is called
            self._new_LR = lr = self.opt_kwargs.pop("learning_rate", 0.2)
            self.optimizer = optim.Momentum(self.arena, lr=lr, decay_rate=self.opt_kwargs.pop("decay_rate", 0.95),
                                            momentum=self.opt_kwargs.pop("momentum", 0.2), weight_decay=self.net.weight_decay_table(tv))
        else:
            lr = self.opt_kwargs.pop("learning_rate", 1e-3)
            self._new_LR = lr
            self.optimizer = optim.Adam(self.arena, lr=lr, weight_decay=self.net.weight_decay_table(tv), **self.opt_kwargs)
        dev = self.arena.theta.device
        self._g_cross = torch.tensor(float(self.net.miu_cross or 0.0) if self.net.cross_flag else 0.0, device=dev)
        self._g_dice = torch.tensor(float(self.net.miu_dice or 0.0) if self.net.dice_flag else 0.0, device=dev)

    def train_step(self, batch_x, batch_y, keep_prob=0.75):
        """one sess.run((optimizer, cost, lr)) of source_segmenter.py:484-489 (both BN switches True).
        batch_x [B,256,256,3] fp32, batch_y [B,256,256,num_cls] one-hot fp32, both on the device."""
        self.arena.zero_grad()
        rt.rng.advance()
        rt.scratch.begin_step()
        logits = self.net.forward(batch_x, keep_prob=keep_prob, main_bn=True, adapt_bn=True)
        wce, dice = self.net.losses(logits, batch_y)
        self.dp.begin_backward(self.arena)
        torch.autograd.backward([wce, dice], [self._g_cross, self._g_dice])
        scale = self.dp.finish_backward(self.arena)
        self.optimizer.step(grad_scale=scale)
        if self.ema is not None:
            self.ema.update()
        self.global_step += 1
        return wce, dice

    def capture_train_step(self, x_example, y_example, keep_prob=0.75, warmup=2):
        """the Adam step as ONE CUDA graph on static input buffers (the warm-up steps are real steps).  The losses are handed out
        detached, for the reason given in Full_DRN.losses: a later capture must not inherit this one's gradient accumulators."""
        self._graph = None
        self._graph = rt.capture_step("segmenter", lambda x, y: self.train_step(x, y, keep_prob), (x_example, y_example),
                                      keep_prob, warmup, self.trainables, (self.arena,), detach=True)
        return self._graph is not None

    def release_graphs(self):
        self._graph = None

    def recalibrate_bn(self, source, batches):
        """re-estimate every batch norm's moving statistics (all 30) as exact population statistics (bnstats.py; DESIGN 6.1)
        over `batches` forwards on images from `source` (.next() -> (images, labels), labels ignored; the network's batch
        size): keep_prob 1, batch-statistics batch norm.  Captured steps are released.  -> (covered variable names, slice
        count).  ValueError: batches < 1 or a wrong batch size; NotImplementedError under data parallelism."""
        from . import bnstats
        covered = bnstats.covered_statistics([v for v in rt.global_variables() if v.pnp_kind == "bn_moving"])
        fwd = lambda x: self.net.forward(x, 1.0, main_bn=True, adapt_bn=True)
        return bnstats.recalibrate(self, source, batches, covered, fwd)

    def entropy_adaptation(self, lr=1e-4):
        """an open tent.EntropyAdaptation: gamma and beta of all 30 batch norms train (batch statistics, keep_prob 1) in a fresh
        Adam over the trainer's arena; every convolution weight stays fixed"""
        from . import tent
        covered = [v for v in self.trainables if v.pnp_kind in ("bn_gamma", "bn_beta")]
        fwd = lambda x: self.net.forward(x, 1.0, main_bn=True, adapt_bn=True)
        return tent.EntropyAdaptation(self, self.arena, covered, fwd, lr, self.trainables)

    def adapt_entropy(self, source, steps, lr=1e-4, recalibrate_batches=200):
        """TENT (tent.py; DESIGN 6.1): `steps` entropy-minimisation steps of every batch norm's gamma / beta on unlabelled images
        from `source` (.next() -> (images, labels), labels ignored; the network's batch size), then recalibrate_bn(source,
        recalibrate_batches).  The trainer's own optimizer and global_step are untouched; anything raising puts the snapshotted
        variables back.  -> (covered variable names, history [steps, 1 + C] numpy, slice count).  ValueError: steps < 1,
        recalibrate_batches < 1, a non-positive lr or a wrong batch size; FloatingPointError: a non-finite loss;
        NotImplementedError under data parallelism."""
        from . import tent
        return tent.adapt(self.entropy_adaptation, source, steps, lr, recalibrate_batches, self.recalibrate_bn)

    def train_step_replay(self, batch_x, batch_y, keep_prob=0.75):
        if not rt.StepGraph.fits(self._graph, keep_prob):
            return self.train_step(batch_x, batch_y, keep_prob)
        self.global_step += 1
        return self._graph.replay(batch_x, batch_y)

    # scalar tags of the merged summary op, in its order (source_segmenter.py:387-396)
    SCALAR_TAGS = ("loss", "regularizer_loss", "weighted_loss", "dice_loss", "dice_eval", "dice_eval_c1", "dice_eval_c2", "dice_eval_c3",
                   "dice_eval_c4")
    # image summaries of the two merged image ops, in their order (source_segmenter.py:398-405): [compact_pred, x[:,:,:,1], compact_y].
    # The validation list's 'image' is the graph's second summary of that name, so its name scope (= tag) is uniquified to 'image_1'
    TRAIN_IMAGE_TAGS = ("train_pred", "image", "GND")
    VAL_IMAGE_TAGS = ("val_pred", "image_1", "validation_GND")

    def _scalars(self, logits, batch_y, wce, dice):
        d, arr = self.net.dice_eval(logits, batch_y)
        vals = [self.net.cost_value(wce, dice), self.net.regularizer_loss(), float(wce), float(dice), float(d)] + \
               [float(arr[i]) for i in range(1, 5)]
        return dict(zip(self.SCALAR_TAGS, vals))

    def _summaries(self, log_dir, step, names, image_summaries, logits, batch_x, batch_y, wce, dice):
        """tf.summary.FileWriter(output_path + '/train_log' | '/val_log').add_summary(scalar_summary_op, step) (source_segmenter.py:
        464-465, 537-539, 567-569), and with `image_summaries` add_summary(summary_img, step) of the merged image op `names`,
        rendered from the pass's own tensors -- [compact_pred, x[:,:,:,1], compact_y] (summary.write_pass)"""
        if log_dir is None:
            return
        u8 = None
        if image_summaries and summary.writes(self, log_dir):
            u8 = F.image_summary([(logits, "softmax2_argmax", 0), (batch_x, "channel", 1), (batch_y, "argmax", 0)])
        summary.write_pass(self, log_dir, step, self._scalars(logits, batch_y, wce, dice), names, u8)

    def output_minibatch_stats(self, batch_x, batch_y, step=None, log_dir=None, image_summaries=False):
        """source_segmenter.py:525-539: the tensorboard pass on the training batch feeds x, y and keep_prob 1 ONLY -- both BN
        switches stay at their placeholder default True, so this forward runs batch-statistics BN and (updates_collections=None)
        moves the moving averages once more.  Reproduced because it changes the trained model's moving statistics.  With `log_dir`
        the nine scalar summaries of the reference go to an event file there; `image_summaries` adds the TRAIN_IMAGE_TAGS panels
        of this forward as a second event with the same step."""
        with torch.no_grad():
            logits = self.net.forward(batch_x, keep_prob=1.0, main_bn=True, adapt_bn=True)
            wce, dice = self.net.losses(logits, batch_y)
            self._summaries(log_dir, step, self.TRAIN_IMAGE_TAGS, image_summaries, logits, batch_x, batch_y, wce, dice)
        return self.net.cost_value(wce, dice)

    def feed(self, images, raw_labels):
        """host batch -> device tensors (the feed_dict copy) + on-device one-hot (lib._label_decomp)"""
        dev = rt.device()
        x = to_device(images, dev)
        y = _label_decomp(self.num_cls, to_device(raw_labels, dev))
        return x, y

    def train(self, output_path, restored_path=None, restore=False, training_iters=100, epochs=100, display_step=5, dropout=0.75,
              image_summaries=False):
        """source_segmenter.py:429-525: optimizer steps, the two monitoring passes every `display_step` (training batch with batch-statistics
        BN, then a validation batch in inference mode) with their scalar summaries, checkpoint + LR*0.9.  `image_summaries` also
        writes each pass's image summaries (TRAIN_IMAGE_TAGS / VAL_IMAGE_TAGS) after its scalars."""
        save_path = os.path.join(output_path, "model.cpkt")
        if epochs == 0:
            return save_path
        os.makedirs(output_path, exist_ok=True)
        d = {}
        if restore and restored_path and os.path.exists(os.path.join(restored_path, "latest.npz")):
            self.net.restore(os.path.join(restored_path, "latest.npz"))
            # tf.train.Saver() also brings back the Adam slots, the learning-rate variable and global_step (:398,:446-452)
            d = self.net.last_restored
            self.optimizer.load_slot_state(d)
            if "pnp/learning_rate" in d:
                self.optimizer.set_lr(float(d["pnp/learning_rate"]))
            if "pnp/global_step" in d:
                self.global_step = int(d["pnp/global_step"])
            if self.lr_update_flag:
                self.optimizer.set_lr(self._new_LR)
        elif restore:
            print("Unable to restore, start from beginning")
        self.dp.broadcast_variables(rt.global_variables())
        if self.optimizer_name == "momentum":
            self.optimizer.decay_steps = training_iters
            self.dp.broadcast_params(self.optimizer.accum)
        else:
            self.dp.broadcast_params(self.optimizer.m)
            self.dp.broadcast_params(self.optimizer.v)
        if self.ema is not None and not self.ema.load_state(d):     # a resumed average continues; otherwise it starts here
            self.ema.init_from_live()
        src = pick_source(self.source, self.train_list, self.batch_size, 1234 + self.dp.rank, self.num_cls)
        # the validation queue of source_segmenter.py:325,467 (val_list), else a second synthetic stream
        val_src = pick_source(self.val_source, self.val_list, self.batch_size, 4321 + self.dp.rank, self.num_cls)
        img = {"image_summaries": True} if image_summaries else {}       # the monitoring calls stay as they were when off
        for epoch in range(epochs):
            for step in range(epoch * training_iters, (epoch + 1) * training_iters):
                start = time.time()
                images, raw_y = src.next()
                x, y = self.feed(images, raw_y)
                wce, dice = self.train_step(x, y, dropout)
                if step % display_step == 0:
                    loss = self.output_minibatch_stats(x, y, step, os.path.join(output_path, "train_log"), **img)
                    logging.info("Training at step %s epoch %s , loss is %0.4f" % (step, epoch, loss))
                    logging.info("Time elapsed %s seconds" % (time.time() - start))
                    # source_segmenter.py:498-505: a validation batch right after it, always with the per-organ table
                    vx, vy = self.feed(*val_src.next())
                    self.val_stats(vx, vy, step, os.path.join(output_path, "val_log"), detail=True, **img)
                    if self.ema is not None:
                        self.ema_val_stats(vx, vy, step, os.path.join(output_path, "val_log"))
                if step % self.checkpoint_space == 0 and step > 10000:
                    self.save(save_path, output_path)
                    self.optimizer.set_lr(self.optimizer.get_lr() * 0.9)
        return save_path

    def checkpoint_state(self):
        self.dp.average_moving_stats(rt.global_variables())
        st = rt.state_dict()
        st.update(self.optimizer.slot_state())
        st["pnp/learning_rate"] = np.float32(self.optimizer.get_lr())
        st["pnp/global_step"] = np.int64(self.global_step)
        if self.ema is not None:
            self.ema.average_over_ranks(self.dp)
            st.update(self.ema.state())
        return st

    def save(self, save_path, output_path):
        save_checkpoint(self, save_path, output_path)

    def val_stats(self, batch_x, batch_y, step=None, log_dir=None, detail=False, image_summaries=False):
        """source_segmenter.py:541-570: inference-mode forward (BN moving stats, keep_prob 1) on a validation batch; `detail` prints
        the per-organ Dice / Jaccard table of the batch's confusion matrix; with `log_dir` the scalar summaries go to an event file,
        followed by the VAL_IMAGE_TAGS panels of this forward if `image_summaries`"""
        from .lib import _indicator_eval
        with torch.no_grad():
            logits = self.net.forward(batch_x, keep_prob=1.0, main_bn=False, adapt_bn=False)
            wce, dice = self.net.losses(logits, batch_y)
            d, arr = self.net.dice_eval(logits, batch_y)
            if detail:
                _indicator_eval(self.net.confusion_matrix(logits, batch_y).cpu().numpy())
            self._summaries(log_dir, step, self.VAL_IMAGE_TAGS, image_summaries, logits, batch_x, batch_y, wce, dice)
        return {"loss": self.net.cost_value(wce, dice), "dice_eval": float(d), "dice_arr": [float(a) for a in arr]}

    EMA_TAGS = ("ema_dice_eval", "ema_dice_eval_c1", "ema_dice_eval_c2", "ema_dice_eval_c3", "ema_dice_eval_c4")

    def ema_val_stats(self, batch_x, batch_y, step=None, log_dir=None):
        """val_stats' forward and Dice with the averaged weights swapped in (nothing else runs under the swap) -> the EMA_TAGS
        scalars, written to `log_dir`'s event file with `step` after the pass's own summaries"""
        with self.ema.swapped(), torch.no_grad():
            logits = self.net.forward(batch_x, keep_prob=1.0, main_bn=False, adapt_bn=False)
            d, arr = self.net.dice_eval(logits, batch_y)
            scalars = dict(zip(self.EMA_TAGS, [float(d)] + [float(arr[i]) for i in range(1, 5)]))
        summary.write_pass(self, log_dir, step, scalars)
        return scalars

    # ---- test protocol on NIfTI subjects (source_segmenter.py:572-675) -----------------------------------------------
    def _logits(self, x):
        """the test protocol's forward: keep_prob 1, main_bn / adapt_bn off (the feed of source_segmenter.py:615-617), x [B, 256,
        256, 3] on the device -> logits [B, 256, 256, C]"""
        return self.net.forward(x, keep_prob=1.0, main_bn=False, adapt_bn=False)

    def test_eval_volume(self, raw, raw_y, flip_correction=True):
        """one subject of test_eval: frames in order (see evaluation.subject_batches for the reference's broken loop header)"""
        from . import evaluation
        dice, jac, cm, pred_vol = evaluation.eval_volume(evaluation.predictor(self._logits, self.num_cls), raw, raw_y,
                                                         self.net.batch_size, self.num_cls, flip_correction, False)
        return dice, jac, cm.astype(np.int64), pred_vol

    def test_eval(self, output_path, flip_correction=True, save_result=False, surface_metrics=False, hd_percentile=None):
        """source_segmenter.py:572-632: inference on the (label, image) .nii pairs of test_label_list / test_nii_list; with
        `save_result` the dense predictions and ground truths go to <output_path>/test_pred as .nii.gz.  `surface_metrics` also
        scores every subject by per-organ ASSD / HD on the GPU (evaluation.surface_distances, voxel units), keeps them in
        `self.sample_surface_list`, prints their mean and spread and writes <output_path>/surface.csv; the return value and
        the Dice / Jaccard output are unchanged.  `hd_percentile` q (95: HD95; only with `surface_metrics`, else ValueError) also
        scores the q-th percentile of the pooled surface distances: an `hd_pct` entry per subject, `hd<q>` lines and columns."""
        from . import evaluation
        return evaluation.run_protocol(self, self._logits, self.num_cls, output_path, "test_pred", flip_correction, save_result,
                                       shuffle=False, write_cm=False, surface_metrics=surface_metrics, hd_percentile=hd_percentile)

    def test_native(self, pairs, output_path, hd_percentile=None, largest_component=None, checkpoints=None, tta=None,
                    locate=None):
        """every raw (image, label) pair segmented on its own grid (native.run): writes <output_path>/native_pred/<name>_label.nii.gz
        and native.csv, prints per-organ Dice and ASSD / HD in mm -> per-subject results.  `hd_percentile` q also scores the q-th
        percentile HD in mm (native.csv column <organ>_hd<q>_mm).  `largest_component` 6 or 26 keeps only the largest connected
        component of each organ before scoring and writing.  `checkpoints` (.npz paths, each restored before its members' frames
        are predicted) and `tta` ((theta_deg, scale_r, scale_c, shift_r, shift_c) test-time transforms) ensemble the prediction
        (native.Ensemble); every variable holds its value from before the call again when it returns.  `locate` (a
        localise.Calibration or its JSON path) crops every subject at the heart box the network locates without its labels."""
        from . import native
        # restore loads exact variable names only
        ensemble = native.trainer_ensemble(self.net, checkpoints, tta, native.SLOT_KEYWORDS, strip_suffix=False)
        return native.run(self._logits, pairs, output_path, self.net.batch_size, self.num_cls, hd_percentile, largest_component,
                          ensemble, locate)

    def segment_native(self, images, output_path, calibration, largest_component=None, checkpoints=None, tta=None):
        """unlabelled scans located with `calibration` and segmented on their own grid (native.segment): writes
        <output_path>/native_pred/<name>_label.nii.gz and located.csv; `largest_component`, `checkpoints` and `tta` as
        test_native takes them"""
        from . import native
        ensemble = native.trainer_ensemble(self.net, checkpoints, tta, native.SLOT_KEYWORDS, strip_suffix=False)
        return native.segment(self._logits, images, output_path, self.net.batch_size, self.num_cls, calibration,
                              largest_component, ensemble)

    def sample_metric_stddev(self, sample_eval_list):
        """source_segmenter.py:634-664"""
        from . import evaluation
        return evaluation.sample_metric_stddev(sample_eval_list, self.num_cls)

    def test_choose_model(self, this_model, output_path, surface_metrics=False, hd_percentile=None):
        """source_segmenter.py:666-675: restore a checkpoint, run the test protocol"""
        self.net.restore(this_model)
        logging.info("model has been loaded!")
        dice, jac = self.test_eval(output_path, surface_metrics=surface_metrics, hd_percentile=hd_percentile)
        logging.info("testing finished")
        return dice, jac
