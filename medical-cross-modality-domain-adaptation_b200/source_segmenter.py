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
from .data import SyntheticSource, to_device
from .lib import _label_decomp, _save
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
        self.weighted_loss, self.dice_loss = wce, dice
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
                 val_source=None):
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
        self._build_optimizer()

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
        self.global_step += 1
        return wce, dice

    def capture_train_step(self, x_example, y_example, keep_prob=0.75, warmup=2):
        """the Adam step as ONE CUDA graph on static input buffers (the warm-up steps are real steps)"""
        self._gx, self._gy = x_example.clone(), y_example.clone()
        self._graph = None
        try:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(warmup):
                    self.train_step(self._gx, self._gy, keep_prob)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            for v in self.trainables:          # see adversarial.Trainer._capture: no stale operand caches inside the graph
                v.__dict__.pop("_pnp_planes", None)
                v.__dict__.pop("_pnp_wT", None)
                v.__dict__.pop("_pnp_bncoef", None)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = self.train_step(self._gx, self._gy, keep_prob)
            self._graph, self._graph_out, self._graph_kp = g, out, keep_prob
            return True
        except Exception as e:      # noqa: BLE001
            import warnings
            warnings.warn("CUDA-graph capture of the segmenter step failed (%s: %s); running eagerly" % (type(e).__name__, e))
            torch.cuda.synchronize()
            self._graph = None
            return False

    def train_step_replay(self, batch_x, batch_y, keep_prob=0.75):
        if getattr(self, "_graph", None) is None or keep_prob != self._graph_kp:
            return self.train_step(batch_x, batch_y, keep_prob)
        self._gx.copy_(batch_x, non_blocking=True)
        self._gy.copy_(batch_y, non_blocking=True)
        self._graph.replay()
        self.global_step += 1
        self.arena.bump_versions()
        return self._graph_out

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

    def _write_scalars(self, log_dir, step, scalars, images=None):
        """tf.summary.FileWriter(output_path + '/train_log' | '/val_log').add_summary(scalar_summary_op, step) (source_segmenter.py:
        464-465, 537-539, 567-569): a TensorBoard event file plus the same numbers as one JSON line; rank 0 only.  `images`
        (tag, uint8 panel) pairs follow as a second event with the same step, as add_summary(summary_img, step) does"""
        if log_dir is None or self.dp.rank != 0:
            return
        import json
        from .summary import FileWriter
        writers = self.__dict__.setdefault("_summary_writers", {})
        if log_dir not in writers:
            writers[log_dir] = FileWriter(log_dir)
        writers[log_dir].add_scalars(scalars, step)
        if images is not None:
            writers[log_dir].add_images(images, step)
        writers[log_dir].flush()
        with open(os.path.join(log_dir, "scalars.jsonl"), "a") as f:
            f.write(json.dumps(dict(step=int(step), **scalars)) + "\n")

    def _images(self, log_dir, names, logits, batch_x, batch_y):
        """the panels of one merged image op from the pass's own tensors -- [compact_pred, x[:,:,:,1], compact_y] -- as
        (tag, uint8 [H, W]) pairs in the merged op's order; None where nothing is written (no log_dir, or not rank 0)"""
        if log_dir is None or self.dp.rank != 0:
            return None
        from .summary import image_tags
        u8 = F.image_summary([(logits, "softmax2_argmax", 0), (batch_x, "channel", 1), (batch_y, "argmax", 0)])
        return [(tag, u8[s, i]) for s, name in enumerate(names) for i, tag in enumerate(image_tags(name, u8.shape[1]))]

    def output_minibatch_stats(self, batch_x, batch_y, step=None, log_dir=None, image_summaries=False):
        """source_segmenter.py:525-539: the tensorboard pass on the training batch feeds x, y and keep_prob 1 ONLY -- both BN
        switches stay at their placeholder default True, so this forward runs batch-statistics BN and (updates_collections=None)
        moves the moving averages once more.  Reproduced because it changes the trained model's moving statistics.  With `log_dir`
        the nine scalar summaries of the reference go to an event file there; `image_summaries` adds the TRAIN_IMAGE_TAGS panels
        of this forward as a second event with the same step."""
        with torch.no_grad():
            logits = self.net.forward(batch_x, keep_prob=1.0, main_bn=True, adapt_bn=True)
            wce, dice = self.net.losses(logits, batch_y)
            if log_dir is not None:
                images = self._images(log_dir, self.TRAIN_IMAGE_TAGS, logits, batch_x, batch_y) if image_summaries else None
                self._write_scalars(log_dir, step, self._scalars(logits, batch_y, wce, dice), images)
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
        if self.source is not None:
            src = self.source
        elif self.train_list:      # the reference's lists/*_train_list of single-example TFRecord files
            from .tfrecord import TFRecordSource
            src = TFRecordSource(self.train_list, self.batch_size, seed=1234 + self.dp.rank)
        else:
            src = SyntheticSource(self.batch_size, seed=1234 + self.dp.rank, num_cls=self.num_cls)
        # the validation queue of source_segmenter.py:325,467 (val_list), else a second synthetic stream
        if self.val_source is not None:
            val_src = self.val_source
        elif self.val_list:
            from .tfrecord import TFRecordSource
            val_src = TFRecordSource(self.val_list, self.batch_size, seed=4321 + self.dp.rank)
        else:
            val_src = SyntheticSource(self.batch_size, seed=4321 + self.dp.rank, num_cls=self.num_cls)
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
        return st

    def save(self, save_path, output_path):
        st = self.checkpoint_state()
        def write():
            _save(st, save_path, global_step=self.global_step)
            _save(st, os.path.join(output_path, "latest"))
        self.dp.save_checkpoint(write)

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
            if log_dir is not None:
                images = self._images(log_dir, self.VAL_IMAGE_TAGS, logits, batch_x, batch_y) if image_summaries else None
                self._write_scalars(log_dir, step, self._scalars(logits, batch_y, wce, dice), images)
        return {"loss": self.net.cost_value(wce, dice), "dice_eval": float(d), "dice_arr": [float(a) for a in arr]}

    # ---- test protocol on NIfTI subjects (source_segmenter.py:572-675) -----------------------------------------------
    def _predict(self, vol, sl):
        """one forward call of the test protocol: keep_prob 1, main_bn / adapt_bn off (the feed of source_segmenter.py:615-617)
        -> (argmax labels, confusion counts [label, prediction]) on the host"""
        dev = rt.device()
        x = torch.from_numpy(np.ascontiguousarray(vol, np.float32)).to(dev)
        y = _label_decomp(self.num_cls, torch.from_numpy(np.ascontiguousarray(sl, np.int64)).to(dev))
        with torch.no_grad():
            logits = self.net.forward(x, keep_prob=1.0, main_bn=False, adapt_bn=False)
            cm = self.net.confusion_matrix(logits, y)
            pred = logits.argmax(3)
        return pred.cpu().numpy(), cm.cpu().numpy()

    def test_eval_volume(self, raw, raw_y, flip_correction=True):
        """one subject of test_eval: frames in order (see evaluation.subject_batches for the reference's broken loop header)"""
        from . import evaluation
        dice, jac, cm, pred_vol = evaluation.eval_volume(self._predict, raw, raw_y, self.net.batch_size, self.num_cls,
                                                         flip_correction, False)
        return dice, jac, cm.astype(np.int64), pred_vol

    def test_eval(self, output_path, flip_correction=True, save_result=False):
        """source_segmenter.py:572-632: inference on the (label, image) .nii pairs of test_label_list / test_nii_list; with
        `save_result` the dense predictions and ground truths go to <output_path>/test_pred as .nii.gz"""
        from . import evaluation
        sample_eval_list, _ = evaluation.run_test_eval(self._predict, self.test_label_list, self.test_nii_list, self.net.batch_size,
                                                       self.num_cls, output_path, "test_pred", flip_correction, save_result,
                                                       shuffle=False, write_cm=False)
        self.sample_eval_list = sample_eval_list
        return self.sample_metric_stddev(sample_eval_list)

    def sample_metric_stddev(self, sample_eval_list):
        """source_segmenter.py:634-664"""
        from . import evaluation
        return evaluation.sample_metric_stddev(sample_eval_list, self.num_cls)

    def test_choose_model(self, this_model, output_path):
        """source_segmenter.py:666-675: restore a checkpoint, run the test protocol"""
        self.net.restore(this_model)
        logging.info("model has been loaded!")
        dice, jac = self.test_eval(output_path)
        logging.info("testing finished")
        return dice, jac
