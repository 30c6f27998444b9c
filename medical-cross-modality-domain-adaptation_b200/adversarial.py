"""PnP-AdaNet adversarial graph and its alternating D / G training steps -- the H100-native counterpart
of the reference's adversarial.py (Full_DRN :44-574, Trainer :576-1108), eager instead of TF-1 graph.

    MR stream : group_1..6 (frozen source segmenter front, BN scopes pred_*)      adversarial.py:130-199
    CT stream : adapt_1..6 (domain adaptation module "DAM", BN scopes adapt_*)      adversarial.py:201-269
    shared    : group_7..10 + output (frozen back half)                              adversarial.py:273-318
    D         : cls_scope  -- multi-scale feature-map discriminator                  adversarial.py:320-400
    M         : mask_cls_scope -- segmentation-mask critic                            adversarial.py:402-443
    losses    : WGAN critic means + L2 regularisers                                   adversarial.py:445-476
    steps     : RMSProp(cls_vars) + clip +-0.03 ; RMSProp(adapt_vars)                 adversarial.py:633-656,840-882

Reference defects reproduced or fixed (SURVEY App. C): `predictor`/`predicter` both exposed; critics
run with hard-wired keep_prob=0.75 and batch-statistics BN (overridable for parity runs); every critic
weight is counted twice in the L2 sums because create_classifier/create_mask_critic append to the weight
lists on each of their two calls.
"""
import logging
import os
import time

import numpy as np
import torch

from . import functional as F
from . import layers as L
from . import optim
from . import parallel
from . import runtime as rt
from .data import SyntheticSource, to_device
from .lib import _save
from .networks import FB, FRONT, BACK, SegmenterHalf, SegmenterTail

# feature discriminator stages: (scope, cin, cout, inc_dim, down kernel, down stride)  adversarial.py:337-386
_CLS_STAGES = [("cls_1", 2 * FB, 4 * FB, True, 3, 2), ("cls_2", 4 * FB, 8 * FB, True, 5, 2), ("cls_3", 8 * FB, 16 * FB, True, 3, 2),
               ("cls_4", 16 * FB, 32 * FB, True, 3, 2), ("cls_5", 32 * FB, 32 * FB, False, 5, 4)]


def _pred_namer(gi, blk, kind):
    base = "pred_%d_%d" % (gi, blk)
    return base if kind == "b" else (base + "_1", base + "_2")


def _adapt_namer(gi, blk, kind):
    # adversarial.py:206-267: scope 'adapt_1' / 'adapt_2' for groups 1-2, 'adapt_k_b' afterwards
    base = "adapt_%d" % gi if gi <= 2 else "adapt_%d_%d" % (gi, blk)
    return (base + "_1", base + "_2")


class Full_DRN(object):

    def __init__(self, channels, n_class, batch_size, cost_kwargs={}, network_config={}, critic_keep_prob=0.75, **kwargs):
        rt.reset_default_graph()
        self.n_class = n_class
        self.batch_size = batch_size
        self.network_config = network_config
        self.mr_front_trainable = network_config.get("mr_front_trainable", False)
        self.ct_front_trainable = network_config.get("ct_front_trainable", True)
        self.joint_trainable = network_config.get("joint_trainable", False)
        self.cls_trainable = network_config.get("cls_trainable", True)
        self.m_cls_trainable = network_config.get("m_cls_trainable", True)
        # hard-wired Python defaults of create_classifier / create_mask_critic (adversarial.py:320,402)
        self.critic_keep_prob = critic_keep_prob
        sd_plain = kwargs.get("stddev_plain", 0.01)    # weight_variable        (groups 1-4 of the MR path)
        sd_share = kwargs.get("stddev", 0.1)           # sharable_weight_variable (everything else)

        self.mr_front_a = SegmenterHalf({g: FRONT[g] for g in (1, 2, 3, 4)}, "group_%d", channels, _pred_namer,
                                        self.mr_front_trainable, sd_plain)
        self.mr_front_b = SegmenterHalf({g: FRONT[g] for g in (5, 6)}, "group_%d", self.mr_front_a.out_channels, _pred_namer,
                                        self.mr_front_trainable, sd_share)
        self.back = SegmenterHalf(BACK, "group_%d", self.mr_front_b.out_channels, _pred_namer, self.joint_trainable, sd_share)
        self.tail = SegmenterTail(n_class, self.joint_trainable, sd_share)
        self.ct_front = SegmenterHalf(FRONT, "adapt_%d", channels, _adapt_namer, self.ct_front_trainable, sd_share)

        # weight lists exactly as the reference fills them (used for the L2 terms, adversarial.py:463-470)
        back_ws = self.back.weights + [self.tail.w10]
        self.mr_front_weights = self.mr_front_a.weights + self.mr_front_b.weights + back_ws + back_ws
        self.ct_front_weights = list(self.ct_front.weights)
        self.joint_weights = []
        self.cls_weights_unique, self.m_cls_weights_unique = self._build_critics(sd_share)
        self.cls_weights = self.cls_weights_unique * 2        # appended on each of the two create_classifier calls
        self.m_cls_weights = self.m_cls_weights_unique * 2

        ck = dict(cost_kwargs)
        self.miu_dis = ck["miu_dis"]
        self.miu_gen = ck["miu_gen"]
        lam = ck.pop("lambda_mask_loss", 1.0)
        self.lambda_mask_loss = 1.0 if lam is None else lam
        self.reg_coeff = ck.pop("regularizer", 1.0e-4)
        self.gan_reg_coeff = ck.pop("gan_regularizer", 1.0e-4)
        self._get_variables_by_scope()

    # ---- variable creation for the critics ---------------------------------------------------------------
    def _build_critics(self, sd):
        cls_w, m_w = [], []
        with rt.variable_scope("cls_scope"):
            for name, cin, cout, inc, dk, ds in _CLS_STAGES:
                with rt.variable_scope(name):
                    cls_w.append(L.sharable_weight_variable([3, 3, cin, cout], sd, self.cls_trainable, "Variable"))
                    cls_w.append(L.sharable_weight_variable([3, 3, cout, cout], sd, self.cls_trainable, "Variable_1"))
                    cls_w.append(L.sharable_weight_variable([dk, dk, cout, cout], sd, self.cls_trainable, "Variable_2"))
                    for sfx in ("_1", "_2", "_3"):
                        L.bn_variables(name + sfx, cout, self.cls_trainable)
            with rt.variable_scope("cls_6"):
                cls_w.append(L.sharable_weight_variable([3, 3, 32 * FB, 32 * FB], sd, self.cls_trainable, "Variable"))
                L.bn_variables("cls_6", 32 * FB, self.cls_trainable)
            with rt.variable_scope("cls_out"):
                cls_w.append(L.sharable_weight_variable([32 * FB * 4, 1], sd, self.cls_trainable, "Variable"))
        t = self.m_cls_trainable
        nc = self.n_class
        with rt.variable_scope("mask_cls_scope"):
            with rt.variable_scope("mask_cls_1"):
                m_w.append(L.sharable_weight_variable([3, 3, nc, FB], sd, t, "Variable"))
                L.bn_variables("mask_cls_1", FB, t)
            with rt.variable_scope("mask_cls_2"):
                m_w.append(L.sharable_weight_variable([3, 3, FB, FB], sd, t, "Variable"))
                m_w.append(L.sharable_weight_variable([3, 3, FB, FB], sd, t, "Variable_1"))
                m_w.append(L.sharable_weight_variable([5, 5, FB, 2 * FB], sd, t, "Variable_2"))
                for sfx, c in (("_1", FB), ("_2", FB), ("_3", 2 * FB)):
                    L.bn_variables("m_cls_2" + sfx, c, t)
            with rt.variable_scope("mask_cls_3"):
                m_w.append(L.sharable_weight_variable([3, 3, 2 * FB, 4 * FB], sd, t, "Variable"))
                m_w.append(L.sharable_weight_variable([3, 3, 4 * FB, 4 * FB], sd, t, "Variable_1"))
                m_w.append(L.sharable_weight_variable([5, 5, 4 * FB, 8 * FB], sd, t, "Variable_2"))
                for sfx, c in (("_1", 4 * FB), ("_2", 4 * FB), ("_3", 8 * FB)):
                    L.bn_variables("m_cls_3" + sfx, c, t)
            with rt.variable_scope("mask_cls_4"):
                m_w.append(L.sharable_weight_variable([5, 5, 8 * FB, 16 * FB], sd, t, "Variable"))
                L.bn_variables("m_cls_4", 16 * FB, t)
            with rt.variable_scope("m_cls_out"):
                m_w.append(L.sharable_weight_variable([16 * FB * 4, 1], sd, t, "Variable"))
        return cls_w, m_w

    def _get_variables_by_scope(self):
        """adversarial.py:478-501: membership by substring of the variable name"""
        self.adapt_vars, self.cls_vars, self.seg_vars, self.mri_seg_vars = [], [], [], []
        for name in rt.graph.order:
            v = rt.graph.vars[name]
            if "cls" in name:
                self.cls_vars.append(v)
            elif "adapt" in name:
                self.adapt_vars.append(v)
            elif "output" in name:
                self.seg_vars.append(v)
                self.mri_seg_vars.append(v)
            elif "group" in name:
                self.mri_seg_vars.append(v)

    # ---- sub-graphs ------------------------------------------------------------------------------------------
    def segment(self, x, stream, keep_prob, front_bn, joint_bn=False):
        """create_zip_network + create_second_half for one stream ('mr' | 'ct')"""
        if stream == "mr":
            h, ta = self.mr_front_a.run(x, keep_prob, front_bn, self.mr_front_trainable)
            h, tb = self.mr_front_b.run(h, keep_prob, front_bn, self.mr_front_trainable)
            c4, c6 = ta[4], tb[6]
        else:
            h, t = self.ct_front.run(x, keep_prob, front_bn, self.ct_front_trainable)
            c4, c6 = t[4], t[6]
        h, t3 = self.back.run(h, keep_prob, joint_bn, self.joint_trainable)
        logits = self.tail.run(h, keep_prob, self.batch_size)
        return {"c4_2": c4, "c6_2": c6, "b7": t3[7], "b8": t3[8], "c9_2": t3[9], "logits": logits}

    def create_classifier(self, input_conv4, input_conv6, input_b7, input_conv9, seg_logits, keep_prob=None, cls_bn=True):
        """adversarial.py:320-400 -> [B,1] critic logits"""
        kp = self.critic_keep_prob if keep_prob is None else keep_prob
        tr = self.cls_trainable
        with rt.variable_scope("cls_scope"):
            h = F.disc_input(input_conv4, input_conv6, input_b7, input_conv9, seg_logits, self.batch_size)
            v = rt.graph.vars
            for name, cin, cout, inc, dk, ds in _CLS_STAGES:
                with rt.variable_scope(name):
                    p = "cls_scope/%s/" % name
                    h = L.residual_block(h, v[p + "Variable"], v[p + "Variable_1"], keep_prob=kp, inc_dim=inc, is_train=cls_bn,
                                         bn_trainable=tr, scope=name, leak=True)
                    h = L.conv_bn_relu2d(h, v[p + "Variable_2"], kp, strides=[1, ds, ds, 1], is_train=cls_bn, bn_trainable=tr,
                                         scope=name + "_3", leak=True)
            with rt.variable_scope("cls_6"):
                h = L.conv_bn_relu2d(h, v["cls_scope/cls_6/Variable"], strides=[1, 2, 2, 1], keep_prob=kp, padding="SYMMETRIC",
                                     scope="cls_6", is_train=cls_bn, bn_trainable=tr, leak=True)
            flat = h.reshape(-1, FB * 32 * 4)
            return F.fc(flat, v["cls_scope/cls_out/Variable"])

    def create_mask_critic(self, input_mask, keep_prob=None, m_cls_bn=True):
        """adversarial.py:402-443 -> [B,1] critic logits"""
        kp = self.critic_keep_prob if keep_prob is None else keep_prob
        tr = self.m_cls_trainable
        v = rt.graph.vars
        m = "mask_cls_scope/"
        with rt.variable_scope("mask_cls_scope"):
            with rt.variable_scope("mask_cls_1"):
                h = L.conv_bn_relu2d(input_mask, v[m + "mask_cls_1/Variable"], kp, strides=[1, 2, 2, 1], is_train=m_cls_bn,
                                     bn_trainable=tr, scope="mask_cls_1", leak=True)
            with rt.variable_scope("mask_cls_2"):
                h = L.residual_block(h, v[m + "mask_cls_2/Variable"], v[m + "mask_cls_2/Variable_1"], keep_prob=kp, inc_dim=False,
                                     is_train=m_cls_bn, bn_trainable=tr, scope="m_cls_2", leak=True)
                h = L.conv_bn_relu2d(h, v[m + "mask_cls_2/Variable_2"], kp, strides=[1, 4, 4, 1], is_train=m_cls_bn,
                                     bn_trainable=tr, scope="m_cls_2_3", leak=True)
            with rt.variable_scope("mask_cls_3"):
                h = L.residual_block(h, v[m + "mask_cls_3/Variable"], v[m + "mask_cls_3/Variable_1"], keep_prob=kp, inc_dim=True,
                                     is_train=m_cls_bn, bn_trainable=tr, scope="m_cls_3", leak=True)
                h = L.conv_bn_relu2d(h, v[m + "mask_cls_3/Variable_2"], kp, strides=[1, 4, 4, 1], is_train=m_cls_bn,
                                     bn_trainable=tr, scope="m_cls_3_3", leak=True)
            with rt.variable_scope("mask_cls_4"):
                h = L.conv_bn_relu2d(h, v[m + "mask_cls_4/Variable"], strides=[1, 4, 4, 1], keep_prob=kp, padding="SYMMETRIC",
                                     scope="m_cls_4", is_train=m_cls_bn, bn_trainable=tr, leak=True)
            flat = h.reshape(-1, FB * 16 * 4)
            return F.fc(flat, v[m + "m_cls_out/Variable"])

    def classify(self, feats):
        return self.create_classifier(feats["c4_2"], feats["c6_2"], feats["b7"], feats["c9_2"], feats["logits"])

    # ---- predictions / metrics ------------------------------------------------------------------------------------
    def predicter(self, logits):
        return L.pixel_wise_softmax_2(logits)

    predictor = predicter   # adversarial.py:101-102 uses both spellings

    def compact_pred(self, logits):
        return torch.argmax(self.predicter(logits), 3)

    def dice_eval(self, logits, y):
        from .lib import _dice_eval
        return _dice_eval(logits, y, self.n_class)

    # ---- losses (adversarial.py:445-476) ------------------------------------------------------------------------------
    def dis_loss_terms(self, ct_cls, mr_cls, ct_mask, mr_mask):
        """returns [(loss tensor, weight in the total)]: dis_loss = -miu*mean(mr-ct) + lambda * (same for masks)"""
        terms = [(F.mean_combo(mr_cls, -self.miu_dis, ct_cls, self.miu_dis), 1.0)]
        if ct_mask is not None:
            terms.append((F.mean_combo(mr_mask, -self.miu_dis, ct_mask, self.miu_dis), self.lambda_mask_loss))
        return terms

    def gen_loss_terms(self, ct_cls, ct_mask):
        terms = [(F.mean_combo(ct_cls, -self.miu_gen), 1.0)]
        if ct_mask is not None:
            terms.append((F.mean_combo(ct_mask, -self.miu_gen), self.lambda_mask_loss))
        return terms

    def dis_reg(self):
        l2 = lambda ws: float(F.l2_loss_sum(ws).item())
        return self.gan_reg_coeff * self.miu_dis * (2 * l2(self.cls_weights_unique) + self.lambda_mask_loss * 2 * l2(self.m_cls_weights_unique))

    def gen_reg(self):
        return self.gan_reg_coeff * self.miu_gen * float(F.l2_loss_sum(self.ct_front_weights).item())

    def fixed_coeff_reg(self):
        """monitoring scalar of adversarial.py:465 (back-half weights counted twice, joint_weights empty)"""
        uniq = self.mr_front_a.weights + self.mr_front_b.weights
        back = self.back.weights + [self.tail.w10]
        return self.reg_coeff * (float(F.l2_loss_sum(uniq).item()) + 2 * float(F.l2_loss_sum(back).item()))

    # ---- checkpoint naming contract (SURVEY 8f #1) --------------------------------------------------------------------------
    def restore(self, model_path, no_gan=False, clear_rms=False, skip_keywords=None):
        """adversarial.py:503-574, on a .npz checkpoint keyed by TF variable names (optimizer slots are never stored).
        no_gan:    only the 'group*' / 'output*' filters of a baseline segmenter checkpoint (no batch norm)   (:514-531)
        clear_rms: every stored variable except the RMSProp slots                                             (:533-550)
        default:   a full restore; if the checkpoint lacks ANY variable of the graph (where tf.train.Saver.restore raises) the
                   relaxed branch loads what is stored except names containing a `restore_skip_kwd` keyword -- the feature
                   discriminator and mask critic ('cls') then start from their initialisation                 (:552-573)"""
        d = dict(np.load(model_path))
        if no_gan:
            # :518-525 -- graph variables present in the checkpoint, minus adapt / cls / Adam names, that contain 'group' or
            # 'output' (a baseline checkpoint names its batch norm 'BatchNorm_k/*', so only the 33 filters qualify; a GAN
            # checkpoint would also hand over its 'group*/pred_*' statistics)
            d = {k: v for k, v in d.items() if k in rt.graph.vars and not any(s_ in k for s_ in ("adapt", "cls", "Adam"))
                 and ("group" in k or "output" in k)}
        elif clear_rms:
            d = {k: v for k, v in d.items() if "RMS" not in k}
        elif any(n not in d for n in rt.graph.order):
            kws = skip_keywords if skip_keywords is not None else self.network_config.get("restore_skip_kwd", ("Adam", "RMS", "cls"))
            d = {k: v for k, v in d.items() if not any(kw in k for kw in kws)}
        self.last_restored = d           # Trainer.train hands the same filtered view to the optimizer slots
        return rt.load_state_dict({k: v for k, v in d.items() if k in rt.graph.vars or (k.endswith(":0") and k[:-2] in rt.graph.vars)},
                                  strict=False)

    def load_batch_norm_weights(self, baseline_path):
        """adversarial.py:743-765: baseline 'BatchNorm_k/*' -> 'group_g/pred_*' in creation order
        (lists/old_bn_list -> lists/pred_bn_list)."""
        d = dict(np.load(baseline_path))
        scopes = []
        for half in (self.mr_front_a, self.mr_front_b, self.back):
            for gi, scope, ops_ in half.plan:
                for op in ops_:
                    if op[0] in ("r", "R", "d"):
                        scopes += [scope + "/" + op[3][0], scope + "/" + op[3][1]]
                    elif op[0] == "b":
                        scopes.append(scope + "/" + op[2])
        out = {}
        for k, s in enumerate(scopes):
            old = "BatchNorm" if k == 0 else "BatchNorm_%d" % k
            for leaf in ("beta", "gamma", "moving_mean", "moving_variance"):
                if old + "/" + leaf in d:
                    out[s + "/" + leaf] = d[old + "/" + leaf]
        return rt.load_state_dict(out, strict=True)

    def adapt_copy_weights(self):
        """adversarial.py:706-741: initialise the CT DAM (adapt_k) from the MR front (group_k), conv weights
        and BN variables, by structural correspondence (lists/half_zip_mri_vars -> lists/half_zip_ct_vars)."""
        src_plan = self.mr_front_a.plan + self.mr_front_b.plan
        with torch.no_grad():
            for (g1, s1, ops1), (g2, s2, ops2) in zip(src_plan, self.ct_front.plan):
                for o1, o2 in zip(ops1, ops2):
                    if o1[0] == "p":
                        continue
                    nw = 1 if o1[0] in ("c", "b") else 2
                    for a, b in zip(o1[1:1 + nw], o2[1:1 + nw]):
                        b.copy_(a)
                        b.pnp_version += 1
                    if o1[0] in ("r", "R", "d"):
                        for sa, sb in zip(o1[3], o2[3]):
                            for leaf in ("beta", "gamma", "moving_mean", "moving_variance"):
                                dst = rt.graph.vars["%s/%s/%s" % (s2, sb, leaf)]
                                dst.copy_(rt.graph.vars["%s/%s/%s" % (s1, sa, leaf)])
                                dst.pnp_version += 1           # cached inference-mode BN coefficients key on the versions


class Trainer(object):
    """adversarial.py:576-1108 re-hosted: alternating D (x dis_sub_iter, + clip) / G (x gen_sub_iter) updates."""

    def __init__(self, net, mr_train_list=None, mr_val_list=None, ct_train_list=None, ct_val_list=None, adapt_var_list=None,
                 mr_var_list=None, old_bn_list=None, new_bn_list=None, test_label_list=None, test_nii_list=None, num_cls=None,
                 batch_size=6, opt_kwargs={}, train_config={}, mr_source=None, ct_source=None):
        self.net = net
        self.batch_size = batch_size
        self.num_cls = num_cls
        self.opt_kwargs = dict(opt_kwargs)
        self.train_config = dict(train_config)
        self.lr_update_flag = self.train_config.get("lr_update", False)
        self.mr_source, self.ct_source = mr_source, ct_source
        self.mr_train_list, self.ct_train_list = mr_train_list, ct_train_list
        self.mr_val_list, self.ct_val_list = mr_val_list, ct_val_list
        self.test_label_list, self.test_nii_list = test_label_list, test_nii_list
        self.dp = parallel.DataParallel()
        self.global_step = 0
        self.dis_sub_iter = self.train_config.get("dis_sub_iter", 1)
        self.gen_sub_iter = self.train_config.get("gen_sub_iter", 1)
        # the objectives `dis_loss + dis_reg / dis_sub_iter` are built once from train_config (adversarial.py:644,650); the
        # schedule's later `dis_sub_iter += dis_sub_iter_inc` (a local of train(), :829/:886) never reaches them
        self._obj_dis_sub_iter, self._obj_gen_sub_iter = self.dis_sub_iter, self.gen_sub_iter
        self._build_optimizers()

    def _build_optimizers(self):
        """adversarial.py:633-656"""
        net = self.net
        lr = self.opt_kwargs.pop("learning_rate", 3e-4)
        self.LR_refresh = lr
        opt = lambda v: getattr(v, "pnp_kind", "") in ("weight", "bn_gamma", "bn_beta")   # moving stats get no gradient
        self.d_vars = [v for v in net.cls_vars if opt(v)]
        self.g_vars = [v for v in net.adapt_vars if opt(v)]
        self.d_arena = optim.Arena(self.d_vars)
        self.g_arena = optim.Arena(self.g_vars)
        # clip_op: every cls var whose name contains "Variable" (conv + FC weights of D and M)
        clip = [0.03 if "Variable" in v.pnp_name else 0.0 for v in self.d_vars]
        self.dp.attach(self.d_arena)
        self.dp.attach(self.g_arena)
        self.dis_optimizer = optim.RMSProp(self.d_arena, lr=lr, clip=clip, **self.opt_kwargs)
        self.gen_optimizer = optim.RMSProp(self.g_arena, lr=lr, **self.opt_kwargs)
        self._refresh_weight_decay()
        self._others = [v for v in rt.global_variables() if id(v) not in {id(x) for x in self.d_vars + self.g_vars}]
        dev = self.d_arena.theta.device
        self._one = torch.tensor(1.0, device=dev)
        self._lam = torch.tensor(float(net.lambda_mask_loss), device=dev)
        self._mode = None

    def _refresh_weight_decay(self):
        """gradient of  dis_reg / dis_sub_iter  and  gen_reg / gen_sub_iter  folded into the optimizer kernels"""
        net = self.net
        d_ids = {id(w) for w in net.cls_weights_unique}
        m_ids = {id(w) for w in net.m_cls_weights_unique}
        base = net.gan_reg_coeff * net.miu_dis * 2.0 / float(self._obj_dis_sub_iter)
        wd = [base if id(v) in d_ids else (base * net.lambda_mask_loss if id(v) in m_ids else 0.0) for v in self.d_vars]
        self.dis_optimizer.set_weight_decay(wd)
        g_ids = {id(w) for w in net.ct_front_weights}
        gb = net.gan_reg_coeff * net.miu_gen / float(self._obj_gen_sub_iter)
        self.gen_optimizer.set_weight_decay([gb if id(v) in g_ids else 0.0 for v in self.g_vars])

    def _set_mode(self, mode):
        """minimize(var_list=...): only the listed variables receive gradients"""
        if self._mode == mode:
            return
        for v in self.d_vars:
            v.requires_grad_(mode == "D")
        for v in self.g_vars:
            v.requires_grad_(mode == "G")
        for v in self._others:
            if v.requires_grad:
                v.requires_grad_(False)
        self._mode = mode

    # ---- the two hot steps --------------------------------------------------------------------------------------------
    def d_step(self, mr_batch, ct_batch, keep_prob=0.75, apply=True):
        """adversarial.py:840-862: feed mr+ct, all segmenter BN switches False, dropout on; dis_optimizer; clip."""
        net = self.net
        self._set_mode("D")
        self.d_arena.zero_grad()
        rt.rng.advance()
        rt.scratch.begin_step()
        with torch.no_grad():
            fm = net.segment(mr_batch, "mr", keep_prob, front_bn=False, joint_bn=False)
            fc_ = net.segment(ct_batch, "ct", keep_prob, front_bn=False, joint_bn=False)
        ct_cls = net.classify(fc_)
        mr_cls = net.classify(fm)
        ct_m = mr_m = None
        if net.lambda_mask_loss != 0:
            ct_m = net.create_mask_critic(fc_["logits"])
            mr_m = net.create_mask_critic(fm["logits"])
        terms = net.dis_loss_terms(ct_cls, mr_cls, ct_m, mr_m)
        self.dp.begin_backward(self.d_arena, overlap=apply)
        torch.autograd.backward([t for t, _ in terms], [self._one, self._lam][:len(terms)])
        if apply:
            self.d_apply()
        return terms

    def d_apply(self):
        """the data-parallel exchange + update of a D step: ONE all-reduce over the gradient arena, then RMSProp + clip"""
        scale = self.dp.finish_backward(self.d_arena)
        self.dis_optimizer.step(grad_scale=scale)
        self.global_step += 1

    def g_step(self, ct_batch, keep_prob=0.75, apply=True):
        """adversarial.py:869-882: feed ct only, ct_front_bn True (DAM BN trains), others False; gen_optimizer."""
        net = self.net
        self._set_mode("G")
        self.g_arena.zero_grad()
        rt.rng.advance()
        rt.scratch.begin_step()
        fc_ = net.segment(ct_batch, "ct", keep_prob, front_bn=True, joint_bn=False)
        ct_cls = net.classify(fc_)
        ct_m = net.create_mask_critic(fc_["logits"]) if net.lambda_mask_loss != 0 else None
        terms = net.gen_loss_terms(ct_cls, ct_m)
        self.dp.begin_backward(self.g_arena, overlap=apply)
        torch.autograd.backward([t for t, _ in terms], [self._one, self._lam][:len(terms)])
        if apply:
            self.g_apply()
        return terms

    def g_apply(self):
        scale = self.dp.finish_backward(self.g_arena)
        self.gen_optimizer.step(grad_scale=scale)
        self.global_step += 1

    def evaluate(self, ct_batch, ct_labels_onehot):
        """adversarial.py:894-922 (CT validation statistics): inference-mode forward of the adapted segmenter (DAM + shared back
        half, moving-statistics BN, keep_prob 1) -> hard Dice (background included) and the confusion matrix"""
        with torch.no_grad():
            out = self.net.segment(ct_batch, "ct", 1.0, front_bn=False, joint_bn=False)
            dice, arr = self.net.dice_eval(out["logits"], ct_labels_onehot)
            cm = F.confusion_counts(out["logits"], ct_labels_onehot)
        return {"dice_eval": float(dice), "dice_arr": [float(a) for a in arr], "confusion_matrix": cm.cpu().numpy()}

    # the reference's TensorBoard scalar tags (adversarial.py:664-683), written as JSON lines because TensorBoard is not a dependency
    SCALAR_TAGS = ("fixed_coeff_reg", "discriminator_loss", "generator_loss", "ct_dice_eval_c1_lv_myo", "ct_dice_eval_c2_la_blood",
                   "ct_dice_eval_c3_lv_blood", "ct_dice_eval_c4_aa", "mri_dice", "learning_rate")
    # image summaries of train_image_summary_op, in its order (adversarial.py:676-682): [compact_pred, ct[:,:,:,1], compact_y,
    # compact_mr_valid, mr[:,:,:,1], compact_mr_y].  output_minibatch_stats fetches this op on every pass, the validation pass
    # (detail=True) included; val_image_summary_op (adversarial.py:684-687, its 'ct_image' uniquified to 'ct_image_1') is built
    # but never fetched, so VAL_IMAGE_TAGS is never written
    TRAIN_IMAGE_TAGS = ("ct_pred", "ct_image", "ct_gt", "mri_validation_pred", "mri_image", "mri_gt")
    VAL_IMAGE_TAGS = ("ct_val_pred", "ct_image_1", "ct_val_gt")

    def output_minibatch_stats(self, step, ct_batch, ct_batch_y, mr_batch, mr_batch_y, log_dir=None, detail=False,
                               image_summaries=False):
        """adversarial.py:948-990, scalar part: one monitoring pass with the segmenter in inference mode and keep_prob 1 (the feed
        also sets cls_bn False, but create_classifier / create_mask_critic never read that placeholder: the critics run with
        their hard-wired batch-statistics BN -- moving averages move -- and keep_prob 0.75, reproduced).  Returns the scalars under
        the reference's tags and appends them to <log_dir>/scalars.jsonl; detail=True also prints per-organ Dice / Jaccard.
        `image_summaries` writes the TRAIN_IMAGE_TAGS panels of this pass's own forwards to the event file after the scalars,
        with the same step (add_summary(summary_str, step); add_summary(summary_img, step))."""
        import json
        from .lib import _indicator_eval
        net = self.net
        rt.scratch.begin_step()
        nc = self.num_cls or net.n_class
        if ct_batch_y.dim() == 3:            # integer label maps: the host-side _label_decomp of the reference, on the device
            ct_batch_y = F.one_hot(ct_batch_y, nc)
        if mr_batch_y.dim() == 3:
            mr_batch_y = F.one_hot(mr_batch_y, nc)
        with torch.no_grad():
            fc_ = net.segment(ct_batch, "ct", 1.0, front_bn=False, joint_bn=False)
            fm = net.segment(mr_batch, "mr", 1.0, front_bn=False, joint_bn=False)
            ct_cls, mr_cls = net.classify(fc_), net.classify(fm)
            ct_m = mr_m = None
            if net.lambda_mask_loss != 0:
                ct_m, mr_m = net.create_mask_critic(fc_["logits"]), net.create_mask_critic(fm["logits"])
            dis = self.loss_value(net.dis_loss_terms(ct_cls, mr_cls, ct_m, mr_m))
            gen = self.loss_value(net.gen_loss_terms(ct_cls, ct_m))
            ct_d, ct_arr = net.dice_eval(fc_["logits"], ct_batch_y)
            mr_d, _ = net.dice_eval(fm["logits"], mr_batch_y)
            cm = F.confusion_counts(fc_["logits"], ct_batch_y) if detail else None
        vals = [net.fixed_coeff_reg(), dis, gen, float(ct_arr[1]), float(ct_arr[2]), float(ct_arr[3]), float(ct_arr[4]), float(mr_d),
                self.dis_optimizer.get_lr()]
        scalars = dict(zip(self.SCALAR_TAGS, vals))
        if detail:
            _indicator_eval(cm.cpu().numpy())
        if log_dir is not None and self.dp.rank == 0:
            # summary_writer.add_summary(summary_str, step); add_summary(summary_img, step); flush() (adversarial.py:989-991): a
            # TensorBoard event file and the same scalars as one JSON line
            from .summary import FileWriter, image_tags
            writers = self.__dict__.setdefault("_summary_writers", {})
            if log_dir not in writers:
                writers[log_dir] = FileWriter(log_dir)
            writers[log_dir].add_scalars(scalars, step)
            if image_summaries:
                u8 = F.image_summary([(fc_["logits"], "softmax2_argmax", 0), (ct_batch, "channel", 1), (ct_batch_y, "argmax", 0),
                                      (fm["logits"], "softmax2_argmax", 0), (mr_batch, "channel", 1), (mr_batch_y, "argmax", 0)])
                writers[log_dir].add_images([(tag, u8[s, i]) for s, name in enumerate(self.TRAIN_IMAGE_TAGS)
                                             for i, tag in enumerate(image_tags(name, u8.shape[1]))], step)
            writers[log_dir].flush()
            with open(os.path.join(log_dir, "scalars.jsonl"), "a") as f:
                f.write(json.dumps(dict(step=int(step), **scalars)) + "\n")
        return scalars

    def _predict_ct(self, vol, sl):
        """one forward call of the test protocol: inference-mode adapted CT stream (keep_prob 1, every BN switch off -- the feed of
        adversarial.py:1036-1038) -> (argmax labels, confusion counts [label, prediction]) on the host"""
        from .lib import _label_decomp
        nc = self.num_cls or self.net.n_class
        dev = rt.device()
        x = torch.from_numpy(np.ascontiguousarray(vol, np.float32)).to(dev)
        y = _label_decomp(nc, torch.from_numpy(np.ascontiguousarray(sl, np.int64)).to(dev))
        with torch.no_grad():
            logits = self.net.segment(x, "ct", 1.0, front_bn=False, joint_bn=False)["logits"]
            cm = F.confusion_counts(logits, y)
            pred = logits.argmax(3)
        return pred.cpu().numpy(), cm.cpu().numpy()

    def test_eval_volume(self, raw, raw_y, flip_correction=True, shuffle_seed=None):
        """adversarial.py:993-1052 for ONE subject: `raw` [256,256,D] intensity volume, `raw_y` [256,256,D] integer labels (what
        read_nii_image returns).  Like the reference: optional flip of both in-plane axes, frames 1..D-2 (each fed with its two
        neighbours as channels) in shuffled order, floor(D / batch) full batches -- the remaining frames are dropped as the
        reference drops them --, inference-mode forward (keep_prob 1, BN switches off), confusion matrix summed over the subject.
        Returns (per-class Dice, per-class Jaccard, confusion matrix, predicted label volume)."""
        from . import evaluation
        rng = None if shuffle_seed is None else np.random.RandomState(shuffle_seed)
        dice, jac, cm, pred_vol = evaluation.eval_volume(self._predict_ct, raw, raw_y, self.net.batch_size,
                                                         self.num_cls or self.net.n_class, flip_correction, True, rng)
        return dice, jac, cm.astype(np.int64), pred_vol

    def test_eval(self, output_path, flip_correction=True, save_result=False, surface_metrics=False):
        """adversarial.py:993-1052: every (label, image) .nii pair of `test_label_list` / `test_nii_list` through the per-subject
        protocol above; writes the summed confusion matrix to <output_path>/cm.csv and returns sample_metric_stddev's pair.
        `save_result` (the segmenter trainer's switch, source_segmenter.py:625-626) also writes the predictions as .nii.gz.
        `surface_metrics` also scores every subject's prediction by per-organ ASSD / HD on the GPU (evaluation.surface_distances,
        voxel units), keeps them in `self.sample_surface_list`, prints their mean and spread and writes
        <output_path>/surface.csv; the return value and the Dice / Jaccard output are unchanged."""
        from . import evaluation
        nc = self.num_cls or self.net.n_class
        res = evaluation.run_test_eval(
            self._predict_ct, self.test_label_list, self.test_nii_list, self.net.batch_size, nc,
            output_path, "dense_pred", flip_correction, save_result, shuffle=True, write_cm=True, surface_metrics=surface_metrics)
        self.sample_eval_list = res[0]
        out = self.sample_metric_stddev(res[0])
        if surface_metrics:
            self.sample_surface_list = res[2]
            evaluation.surface_metric_stddev(res[2], nc)
            evaluation.write_surface_csv(os.path.join(output_path, "surface.csv"), res[2], nc)
        return out

    def sample_metric_stddev(self, sample_eval_list):
        """adversarial.py:1054-1084"""
        from . import evaluation
        return evaluation.sample_metric_stddev(sample_eval_list, self.num_cls or self.net.n_class)

    def test_model(self, this_model, output_path, surface_metrics=False):
        """adversarial.py:1097-1108: restore a checkpoint, run the test protocol"""
        self.net.restore(this_model)
        logging.info("model has been loaded!")
        dice, jac = self.test_eval(output_path, surface_metrics=surface_metrics)
        logging.info("testing finished")
        return dice, jac

    # ---- steps as CUDA graphs -----------------------------------------------------------------------------------------
    def _capture(self, fn, warmup):
        """Capture `fn()` (forward, backward, all-reduce, optimizer, clip: ~1 k kernel launches) into one CUDA graph.
        Dropout seeds, optimizer hyper-state and BN statistics live in device memory, so every replay is a genuinely new
        training step.  Returns (graph, outputs) or (None, None) -- loudly -- if capture fails."""
        try:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(warmup):
                    fn()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            # the per-variable operand caches (bf16 weight planes, transposed SIMT weights) are keyed by a HOST-side version
            # counter: a hit during capture would record no split kernel and freeze the warm-up buffers into the graph, i.e.
            # every replay would run on pre-capture weights.  Drop them so the captured step re-derives them from the live
            # arenas, and keep the variables' versions moving on every replay for eager code that runs later.
            self._invalidate_operand_caches()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = fn()
            return g, out
        except Exception as e:      # noqa: BLE001 -- any capture problem => eager path, loudly
            import warnings
            warnings.warn("CUDA-graph capture of the adversarial step failed (%s: %s); running eagerly" % (type(e).__name__, e))
            torch.cuda.synchronize()
            return None, None

    def capture_joint_step(self, mr_example, ct_example, keep_prob=0.75, warmup=2):
        """`d_step(mr, ct)` + `g_step(ct_g)` as ONE graph on static input buffers (the warm-up steps are real steps)."""
        self._gx_mr, self._gx_ct, self._gx_ct_g = mr_example.clone(), ct_example.clone(), ct_example.clone()
        self._graph, self._graph_out = self._capture(
            lambda: (self.d_step(self._gx_mr, self._gx_ct, keep_prob), self.g_step(self._gx_ct_g, keep_prob)), warmup)
        self._graph_kp = keep_prob
        return self._graph is not None

    def capture_d_step(self, mr_example, ct_example, keep_prob=0.75, warmup=2):
        """the discriminator update alone (pre-train phase; the n_D inner iterations of train-gan)"""
        self._dx_mr, self._dx_ct = mr_example.clone(), ct_example.clone()
        self._d_graph, self._d_graph_out = self._capture(lambda: self.d_step(self._dx_mr, self._dx_ct, keep_prob), warmup)
        self._d_graph_kp = keep_prob
        return self._d_graph is not None

    def capture_g_step(self, ct_example, keep_prob=0.75, warmup=2):
        self._gsx_ct = ct_example.clone()
        self._g_graph, self._g_graph_out = self._capture(lambda: self.g_step(self._gsx_ct, keep_prob), warmup)
        self._g_graph_kp = keep_prob
        return self._g_graph is not None

    def d_step_replay(self, mr_batch, ct_batch, keep_prob=0.75):
        if getattr(self, "_d_graph", None) is None or keep_prob != self._d_graph_kp:
            return self.d_step(mr_batch, ct_batch, keep_prob)
        self._dx_mr.copy_(mr_batch, non_blocking=True)
        self._dx_ct.copy_(ct_batch, non_blocking=True)
        self._d_graph.replay()
        self.global_step += 1
        self.d_arena.bump_versions()
        return self._d_graph_out

    def g_step_replay(self, ct_batch, keep_prob=0.75):
        if getattr(self, "_g_graph", None) is None or keep_prob != self._g_graph_kp:
            return self.g_step(ct_batch, keep_prob)
        self._gsx_ct.copy_(ct_batch, non_blocking=True)
        self._g_graph.replay()
        self.global_step += 1
        self.g_arena.bump_versions()
        return self._g_graph_out

    def release_graphs(self):
        for n in ("_graph", "_graph_out", "_d_graph", "_d_graph_out", "_g_graph", "_g_graph_out"):
            setattr(self, n, None)

    def _invalidate_operand_caches(self):
        for v in self.d_vars + self.g_vars:
            v.__dict__.pop("_pnp_planes", None)
            v.__dict__.pop("_pnp_wT", None)
            v.__dict__.pop("_pnp_bncoef", None)      # inference-mode BN coefficients of the DAM (its statistics move in the G step)

    def joint_step(self, mr_batch, ct_batch, keep_prob=0.75, ct_batch_g=None):
        """one full adversarial step (D update + clip, then G update); replays the captured graph when there is one.
        `ct_batch_g`: the fresh CT batch the reference dequeues for the generator update (adversarial.py:869-873);
        None re-uses the D step's CT batch."""
        if getattr(self, "_graph", None) is not None and keep_prob == self._graph_kp:
            self._gx_mr.copy_(mr_batch, non_blocking=True)
            self._gx_ct.copy_(ct_batch, non_blocking=True)
            self._gx_ct_g.copy_(ct_batch if ct_batch_g is None else ct_batch_g, non_blocking=True)
            self._graph.replay()
            self.global_step += 2
            # the replay changed both arenas on the device: eager code that follows must not trust its cached operands
            self.d_arena.bump_versions()
            self.g_arena.bump_versions()
            return self._graph_out
        return self.d_step(mr_batch, ct_batch, keep_prob), self.g_step(ct_batch if ct_batch_g is None else ct_batch_g, keep_prob)

    # ---- checkpoint contents: tf.train.Saver() stores every global variable -- model variables, both optimizers' slots,
    #      learning_rate_node and global_step (adversarial.py:640,662,929) ---------------------------------------------
    def checkpoint_state(self):
        self.dp.average_moving_stats(rt.global_variables())
        st = rt.state_dict()
        st.update(self.dis_optimizer.slot_state())
        st.update(self.gen_optimizer.slot_state())
        st["pnp/learning_rate"] = np.float32(self.dis_optimizer.get_lr())       # TF names these two scalars 'Variable_k' by
        st["pnp/global_step"] = np.int64(self.global_step)                      # creation order; stable keys here
        return st

    def load_optimizer_state(self, d, clear_rms=False):
        """what a tf.train.Saver restore brings back besides the model: RMSProp slots (unless clear_rms, whose name filter
        'RMS' drops them, :541), the learning-rate variable and global_step"""
        n = 0
        if not clear_rms:
            n = self.dis_optimizer.load_slot_state(d) + self.gen_optimizer.load_slot_state(d)
        if "pnp/learning_rate" in d:
            lr = float(d["pnp/learning_rate"])
            self.dis_optimizer.set_lr(lr)
            self.gen_optimizer.set_lr(lr)
        if "pnp/global_step" in d:
            self.global_step = int(d["pnp/global_step"])
        return n

    def save(self, save_path, output_path):
        st = self.checkpoint_state()
        def write():
            _save(st, save_path, global_step=self.global_step)
            _save(st, os.path.join(output_path, "latest"))
        self.dp.save_checkpoint(write)

    @staticmethod
    def loss_value(terms):
        return sum(float(t.detach()) * w for t, w in terms)

    # ---- schedule (adversarial.py:767-940) ---------------------------------------------------------------------------------
    def train(self, output_path, restore=True, restored_path=None, training_iters=200, epochs=1000, dropout=0.75, display_step=5,
              image_summaries=False):
        """adversarial.py:767-946; `image_summaries` also writes both monitoring passes' image summaries (TRAIN_IMAGE_TAGS)"""
        save_path = os.path.join(output_path, "model.cpkt")
        if epochs == 0:
            return save_path
        os.makedirs(output_path, exist_ok=True)
        cfg = self.train_config
        if restore and restored_path and os.path.exists(os.path.join(restored_path, "latest.npz")):
            ck = os.path.join(restored_path, "latest.npz")
            self.net.restore(ck, no_gan=cfg.get("restore_from_baseline", False), clear_rms=cfg.get("clear_rms", False))
            if cfg.get("restore_from_baseline", False):
                self.net.load_batch_norm_weights(ck)
                print("initializing from baseline model!")
                self.net.adapt_copy_weights()
            else:
                self.load_optimizer_state(self.net.last_restored, clear_rms=cfg.get("clear_rms", False))
        # data parallel: every replica continues from rank 0's variables (weights, frozen parts, BN statistics, slots)
        self.dp.broadcast_variables(rt.global_variables())
        for opt_ in (self.dis_optimizer, self.gen_optimizer):
            self.dp.broadcast_params(opt_.ms)
            self.dp.broadcast_params(opt_.mom)
        if self.lr_update_flag:
            self.dis_optimizer.set_lr(self.LR_refresh)
            self.gen_optimizer.set_lr(self.LR_refresh)
        B = self.batch_size
        def source(given, files, seed, **kw):
            if given is not None:
                return given
            if files:                  # lists/{mr,ct}_train_list: single-example TFRecord files (README.md:49-64)
                from .tfrecord import TFRecordSource
                return TFRecordSource(files, B, seed=seed + self.dp.rank)
            return SyntheticSource(B, seed=seed + self.dp.rank, num_cls=self.num_cls or 5, **kw)
        mr_src = source(self.mr_source, self.mr_train_list, 1234)
        ct_src = source(self.ct_source, self.ct_train_list, 4321, shift=0.3, scale=0.8)
        # the validation queues of adversarial.py:811-815 (lists/{mr,ct}_val_list), else further synthetic streams
        mr_val = source(None, self.mr_val_list, 2234)
        ct_val = source(None, self.ct_val_list, 5321, shift=0.3, scale=0.8)
        dev = rt.device()
        dis_interval, gen_interval = cfg.get("dis_interval", 1), cfg.get("gen_interval", 1)
        dis_inc, gen_inc = cfg.get("dis_sub_iter_inc", 0), cfg.get("gen_sub_iter_inc", 0)
        upd_interval = cfg.get("iter_upd_interval", 999999999999)
        ckpt_space = cfg.get("checkpoint_space", 100)
        decay = cfg.get("lr_decay_factor", 0.98)
        img = {"image_summaries": True} if image_summaries else {}       # the monitoring calls stay as they were when off
        for epoch in range(epochs):
            for step in range(epoch * training_iters, (epoch + 1) * training_iters):
                start = time.time()
                if dis_interval != 0 and step % dis_interval == 0 and step != 0:       # nothing trains at step 0
                    for _ in range(self.dis_sub_iter):
                        ct, _ = ct_src.next()
                        mr, _ = mr_src.next()
                        self.d_step(to_device(mr, dev), to_device(ct, dev), dropout)
                if gen_interval != 0 and step % gen_interval == 0 and step != 0:
                    for _ in range(self.gen_sub_iter):
                        ct, _ = ct_src.next()
                        self.g_step(to_device(ct, dev), dropout)
                if step % upd_interval == 0 and step != 0:
                    self.dis_sub_iter += dis_inc
                    self.gen_sub_iter += gen_inc
                if step % display_step == 0:
                    logging.info("Training step %s epoch %s finished, %.3f s" % (step, epoch, time.time() - start))
                    # the monitoring passes of adversarial.py:894-922: a training batch, then a validation batch with the per-organ table
                    tag = str(self.train_config.get("tag", ""))      # FileWriter(output_path + "/train_log" + tag) (adversarial.py:807-808)
                    for sub, detail, cs, ms in (("train_log", False, ct_src, mr_src), ("val_log", True, ct_val, mr_val)):
                        (ct, cty), (mr, mry) = cs.next(), ms.next()
                        self.output_minibatch_stats(step, to_device(ct, dev), to_device(cty, dev), to_device(mr, dev), to_device(mry, dev),
                                                    os.path.join(output_path, sub + tag), detail, **img)
                if step % ckpt_space == 0 and step != 0:
                    self.save(save_path, output_path)
                    # "Model has been restored for re-allocation" (adversarial.py:929-935): the reference re-reads the checkpoint it
                    # has just written -- numerically a no-op, kept so that a corrupt write surfaces immediately on every rank
                    self.net.restore(os.path.join(output_path, "latest.npz"))
                    self.load_optimizer_state(self.net.last_restored)
                    lr = self.dis_optimizer.get_lr() * decay
                    self.dis_optimizer.set_lr(lr)
                    self.gen_optimizer.set_lr(lr)
        return save_path
