"""Record the REFERENCE'S OWN TensorBoard image-summary wiring -- `Trainer._initialize` and `Trainer.train` of both trainers
(source_segmenter.py:383-570, adversarial.py:658-991), executed unmodified under the recording `tensorflow` shim of
make_reference_graph_trace.py -- and commit it as tests/golden/reference_image_summaries.json.

Recorded:
* every `tf.summary.image` call: its name, which merged op (list) it joins, the provenance of its tensor, whether `max_outputs`
  was passed (the default 3 then applies), and the tag TensorFlow derives for it;
* every monitoring call of the training loops: the step, which merged scalar / image ops the `sess.run` fetches, which writer
  (log directory) then receives which of them through `add_summary`, in order, and the step each is written with.

Restated, not executed: TF-1.4's tag rule.  `tf.summary.image(name, ...)` opens `ops.name_scope(name)`, whose name is made unique
in the graph the way `Graph.unique_name` does it (a repeated name gets `_1`, `_2`, ...), and the uniquified scope is the tag.
ImageSummaryOp then names its values '<tag>/image/<i>' for i < min(batch, max_images), because max_images = 3 > 1.

Only what the image path needs is set up beyond that file's shim: `Full_DRN.__init__` of the GAN stops at adversarial.py:102
(`self.predicter`), so the attributes of adversarial.py:101-115 that the summaries read are assigned as those lines would assign
them (with `predictor`), using the reference's own `pixel_wise_softmax_2`; the data queues (`next_batch`) return zero batches.

    python tests/golden/make_reference_image_summaries.py          # needs the reference sources; the tests only read the .json
"""
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_reference_graph_trace as T  # noqa: E402

OUT = os.path.join(HERE, "reference_image_summaries.json")
BATCH = T.BATCH


class _NullRecorder(object):
    """the layer recorder of the graph trace is not needed here"""

    def raw(self, *a, **k):
        pass

    def _close(self):
        pass

    def set_section(self, name):
        pass

    def emit(self, ev):
        pass


def _getitem(self, idx):
    """Sym.__getitem__ that keeps the index in the provenance (x[:,:,:,1] -> 'ph:x[:,:,:,1]')"""
    idx = idx if isinstance(idx, tuple) else (idx,)
    shape = []
    for n, i in zip(self.shape, idx):
        if isinstance(i, slice):
            shape.append(len(range(*i.indices(n))))
    shape += self.shape[len(idx):]
    txt = ",".join(":" if isinstance(i, slice) and i == slice(None) else repr(i) for i in idx)
    return T.Sym(shape, "%s[%s]" % (self.src, txt))


class Summaries(object):
    """tf.summary: scalar / image / merge / FileWriter, recording"""

    def __init__(self):
        self.used = {}            # name-scope names already taken in this graph
        self.images = []
        self.merged = []
        self.writes = []

    def _scope(self, name):
        n = self.used.get(name, 0)
        self.used[name] = n + 1
        return name if n == 0 else "%s_%d" % (name, n)

    def scalar(self, name, tensor):
        return {"kind": "scalar", "name": name, "tag": self._scope(name)}

    def image(self, name, tensor, max_outputs=None, **kw):
        src = tensor.src if isinstance(tensor, T.Sym) else repr(tensor)
        rec = {"kind": "image", "name": name, "tag": self._scope(name), "tensor": src, "shape": list(tensor.shape),
               "max_outputs_passed": max_outputs is not None, "max_outputs": 3 if max_outputs is None else int(max_outputs)}
        self.images.append(rec)
        return rec

    def merge(self, lst):
        op = "merged_%d" % len(self.merged)
        kinds = sorted({s["kind"] for s in lst})
        self.merged.append({"op": op, "kinds": kinds, "names": [s["name"] for s in lst], "tags": [s["tag"] for s in lst]})
        for s in lst:
            if s["kind"] == "image":
                s.setdefault("lists", []).append(op)
        return op

    def FileWriter(self, logdir, graph=None):
        me = self

        class _W(object):
            def add_summary(self, summary, step):
                me.writes.append({"writer": os.path.basename(os.path.normpath(logdir)), "summary": summary, "step": int(step)})

            def flush(self):
                pass
        return _W()


def _zeros_batch():
    return np.zeros((BATCH, 256, 256, 4), np.float32)


def _monitor(fetches, feeds, S, log):
    fl = list(fetches) if isinstance(fetches, (list, tuple)) else [fetches]
    ops = [f for f in fl if isinstance(f, str) and f.startswith("merged_")]
    if ops:
        log.append({"op": "monitor", "fetch_merged": ops, "feeds": sorted(feeds), "first_write": len(S.writes)})
    return ops


def trace_segmenter(tf):
    """source_segmenter.py: module preamble + Full_DRN + Trainer up to test_eval (the file has a SyntaxError further down), as
    make_reference_graph_trace.trace_source_segmenter executes it"""
    path = os.path.join(T.REF, "source_segmenter.py")
    lines = open(path).read().split("\n")
    cut = next(i for i, ln in enumerate(lines) if ln.strip().startswith("def test_eval"))
    T.G.reset()
    mod = types.ModuleType("pnp_reference_source_segmenter")
    mod.__file__ = path
    exec(compile("\n".join(lines[:cut]) + "\n", path, "exec"), mod.__dict__)
    net = mod.Full_DRN(channels=3, n_class=5, batch_size=BATCH, main_trainable=False, adapt_trainable=True,
                       cost_kwargs={"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0, "regularizer": 1e-4})
    S = Summaries()
    tf.summary = S
    log = []
    names = {id(net.x): "x", id(net.y): "y", id(net.main_bn): "main_bn", id(net.adapt_bn): "adapt_bn", id(net.keep_prob): "keep_prob"}

    class _Feed(object):
        def __init__(self, kind):
            self.kind = kind

        def value(self):
            return _zeros_batch() if self.kind == "data" else [b"file:0"] * BATCH

        def eval(self):
            return self.value()

    class Session(object):
        graph = "graph"

        def __init__(self, config=None):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

        def run(self, fetches, feed_dict=None):
            feeds = {names[id(k)] for k in (feed_dict or {})}
            ops = _monitor(fetches, feeds, S, log)
            fl = list(fetches) if isinstance(fetches, (list, tuple)) else [fetches]
            if fl and fl[0] == "adam_op":
                return None, 0.0, 1e-3
            out = []
            for f in fl:
                if isinstance(f, _Feed):
                    out.append(f.value())
                elif isinstance(f, str) and f in ops:
                    out.append("value_of:" + f)
                elif isinstance(f, T.Sym) and f.src == "cm":
                    out.append(np.zeros((5, 5)))
                else:
                    out.append(0.0)
            return out if isinstance(fetches, (list, tuple)) else out[0]
    tf.Session = Session
    tf.ConfigProto = lambda: types.SimpleNamespace(gpu_options=types.SimpleNamespace(allow_growth=False))

    class AdamOptimizer(object):
        def __init__(self, learning_rate=None, **kw):
            pass

        def minimize(self, loss, global_step=None, var_list=None):
            return "adam_op"
    tf.train = types.ModuleType("tensorflow.train")
    tf.train.AdamOptimizer = AdamOptimizer
    tf.train.string_input_producer = lambda lst, num_epochs=None, shuffle=True: "queue"
    tf.train.Coordinator = lambda: types.SimpleNamespace(request_stop=lambda: None, join=lambda threads: None)
    tf.train.get_checkpoint_state = lambda path: None
    tf.train.start_queue_runners = lambda sess=None, coord=None, start=True: []
    saved_var = tf.Variable

    class _Scalar(float):
        def eval(self):
            return float(self)
    tf.Variable = lambda initial, trainable=True, name=None: (saved_var(initial, trainable, name) if isinstance(initial, T._Init)
                                                               else (_Scalar(initial) if np.isscalar(initial) else "var"))
    tf.assign = lambda var, val: ("assign_lr", float(val))
    tf.global_variables_initializer = lambda: "init_glb"
    tf.variables_initializer = lambda v: "init_loc"
    tf.local_variables = lambda: []
    tf.trainable_variables = lambda: []

    class Me(mod.Trainer):
        def next_batch(self, input_queue, **k):
            return _Feed("data"), _Feed("fid")
    me = Me(net, train_list=["a"], val_list=["b"], num_cls=5, batch_size=BATCH, opt_kwargs={"learning_rate": 1e-3},
            checkpoint_space=1500, optimizer="adam", lr_update_flag=False)
    me.train(output_path="./seg_out", training_iters=7, epochs=1, restore=True, restored_path="./seg_out")
    tf.Variable = saved_var
    return _result(S, log, {"training_iters": 7, "epochs": 1, "display_step": 5})


def trace_gan(tf, adv, layers, mr_logits):
    """adversarial.py: Trainer._initialize + Trainer.train (and output_minibatch_stats) as they are"""
    T.G.reset()
    net = adv.Full_DRN.__new__(adv.Full_DRN)
    cfg = {"mr_front_trainable": False, "ct_front_trainable": True, "joint_trainable": False, "cls_trainable": True, "m_cls_trainable": True,
           "restore_skip_kwd": ["Adam", "RMS", "cls"]}
    cost_kwargs = {"regularizer": 1e-4, "gan_regularizer": 1e-4, "miu_dis": 1e-3, "miu_gen": 2e-3, "lambda_mask_loss": 0.1}
    try:
        adv.Full_DRN.__init__(net, channels=3, n_class=5, batch_size=BATCH, cost_kwargs=cost_kwargs, network_config=cfg)
        raise AssertionError("Full_DRN.__init__ was expected to stop at adversarial.py:102")
    except AttributeError as e:
        assert "predicter" in str(e), e
    # adversarial.py:102-115 as written, with `predictor` (the attribute line 101 did assign)
    net.compact_pred = tf.argmax(net.predictor, 3)
    net.compact_y = tf.argmax(net.ct_y, 3)
    net.mr_seg_valid = layers.pixel_wise_softmax_2(mr_logits[-1])
    net.compact_mr_valid = tf.argmax(net.mr_seg_valid, 3)
    net.compact_mr_y = tf.argmax(net.mr_y, 3)
    for a in ("ct_dice_eval_c1", "ct_dice_eval_c2", "ct_dice_eval_c3", "ct_dice_eval_c4", "mr_dice_eval", "fixed_coeff_reg",
              "confusion_matrix"):
        setattr(net, a, T.Sym([], a))

    class _Loss(object):
        def __add__(self, o):
            return self
        __radd__ = __add__
        __mul__ = __rmul__ = __add__
    net.dis_loss = net.dis_reg = net.ct_gen_loss = net.gen_reg = _Loss()
    tf.contrib.framework.get_variables = lambda: [T._VarObj(T.G.vars[n]) for n in T.G.order]

    S = Summaries()
    tf.summary = S
    log = []
    names = {id(net.mr): "mr", id(net.ct): "ct", id(net.mr_y): "mr_y", id(net.ct_y): "ct_y", id(net.mr_front_bn): "mr_front_bn",
             id(net.joint_bn): "joint_bn", id(net.ct_front_bn): "ct_front_bn", id(net.cls_bn): "cls_bn", id(net.keep_prob): "keep_prob"}

    class _Feed(object):
        def __init__(self, q):
            self.q = q

    class Session(object):
        graph = "graph"

        def __init__(self, config=None):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

        def run(self, fetches, feed_dict=None):
            feeds = {names[id(k)] for k in (feed_dict or {})}
            ops = _monitor(fetches, feeds, S, log)
            fl = list(fetches) if isinstance(fetches, (list, tuple)) else [fetches]
            if fl and fl[0] in ("dis_optimizer", "gen_optimizer"):
                return None, 3e-4
            out = []
            for f in fl:
                if isinstance(f, _Feed):
                    out.append(_zeros_batch() if f.q.endswith("data") else [b"fid"] * BATCH)
                elif isinstance(f, str) and f in ops:
                    out.append("value_of:" + f)
                elif isinstance(f, T.Sym) and f.src == "confusion_matrix":
                    out.append(np.zeros((5, 5)))
                else:
                    out.append(None)
            return out if isinstance(fetches, (list, tuple)) else out[0]
    tf.Session = Session
    tf.ConfigProto = lambda: types.SimpleNamespace(gpu_options=types.SimpleNamespace(allow_growth=False))
    tf.train = types.ModuleType("tensorflow.train")
    tf.train.Coordinator = lambda: types.SimpleNamespace(request_stop=lambda: None, join=lambda threads: None)
    tf.train.get_checkpoint_state = lambda path: None
    tf.train.start_queue_runners = lambda sess=None, coord=None, start=True: []

    class RMSPropOptimizer(object):
        n = 0

        def __init__(self, learning_rate=None, **kw):
            pass

        def minimize(self, loss, global_step=None, var_list=None):
            RMSPropOptimizer.n += 1
            return "dis_optimizer" if RMSPropOptimizer.n == 1 else "gen_optimizer"
    tf.train.RMSPropOptimizer = RMSPropOptimizer
    saved_var, saved_clip = tf.Variable, tf.clip_by_value
    tf.Variable = lambda initial, trainable=True, name=None: (saved_var(initial, trainable, name) if isinstance(initial, T._Init)
                                                               else types.SimpleNamespace(eval=lambda: 0, value=initial))
    tf.clip_by_value = lambda v, lo, hi, name=None: ("clip", v)
    tf.assign = lambda var, val: ("assign", val)
    tf.global_variables_initializer = lambda: "init_glb"
    tf.variables_initializer = lambda v: "init_loc"
    tf.local_variables = lambda: []

    class Me(adv.Trainer):
        def __init__(self):                       # the real one only stores its arguments and opens the input queues
            self.net = net
            self.num_cls = 5
            self.batch_size = BATCH
            self.opt_kwargs = {"learning_rate": 3e-4}
            self.train_config = {"restore_from_baseline": False, "copy_main": False, "clear_rms": False, "lr_update": True,
                                 "dis_interval": 1, "gen_interval": 1, "dis_sub_iter": 1, "gen_sub_iter": 1, "tag": "t",
                                 "checkpoint_space": 100, "lr_decay_factor": 0.98}
            self.lr_update_flag = True
            self.ct_train_queue, self.ct_val_queue, self.mr_train_queue, self.mr_val_queue = "ct_train", "ct_val", "mr_train", "mr_val"

        def next_batch(self, input_queue, **k):
            return _Feed(input_queue + ":data"), _Feed(input_queue + ":fid")
    me = Me()
    me.train(output_path="./gan_out", restore=True, restored_path="./gan_out", training_iters=5, epochs=1, dropout=0.75, display_step=2)
    tf.Variable, tf.clip_by_value = saved_var, saved_clip
    return _result(S, log, {"training_iters": 5, "epochs": 1, "display_step": 2, "tag": "t"})


def _result(S, log, args):
    kinds = {m["op"]: m["kinds"] for m in S.merged}
    for ev in log:
        ev["fetch_kinds"] = [kinds[o] for o in ev["fetch_merged"]]
    return {"image_summaries": S.images, "merged": S.merged, "monitor_calls": log, "writes": S.writes, "loop_args": args}


def main():
    tf, mods = T._make_tf()
    sys.modules.update(mods)
    for name in ("nibabel", "matplotlib"):
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = types.ModuleType(name)
    T.REC = _NullRecorder()
    T.Sym.__getitem__ = _getitem
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp(prefix="pnp_imgsum_"))
    try:
        layers = T._load("layers")
        real_softmax = layers.pixel_wise_softmax_2

        def pixel_wise_softmax_2(output_map):
            out = real_softmax(output_map)
            return T.Sym(out.shape, "pixel_wise_softmax_2(%s)" % output_map.src)
        layers.pixel_wise_softmax_2 = pixel_wise_softmax_2
        T._load("ops")
        T._load("lib")
        adv = T._load("adversarial")
        adv.pixel_wise_softmax_2 = pixel_wise_softmax_2
        mr_logits = []
        real_half = adv.Full_DRN.create_second_half

        def create_second_half(self, *a, **k):
            out = real_half(self, *a, **k)
            mr_logits.append(out[3])
            return out
        adv.Full_DRN.create_second_half = create_second_half
        gan = trace_gan(tf, adv, layers, mr_logits)
        sys.modules["layers"].pixel_wise_softmax_2 = pixel_wise_softmax_2
        seg = trace_segmenter(tf)
    finally:
        os.chdir(cwd)
    rec = {"batch": BATCH, "source_segmenter": seg, "adversarial": gan,
           "tag_rule": "TF-1.4 (restated): tag = name_scope(name) uniquified as Graph.unique_name; values '<tag>/image/<i>', "
                       "i < min(batch, max_outputs)"}
    with open(OUT, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
    print("wrote %s: %d + %d image summaries, %d + %d monitoring calls" % (OUT, len(seg["image_summaries"]), len(gan["image_summaries"]),
                                                                          len(seg["monitor_calls"]), len(gan["monitor_calls"])))


if __name__ == "__main__":
    main()
