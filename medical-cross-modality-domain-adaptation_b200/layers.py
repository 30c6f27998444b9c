"""Operator surface of the reference's layers.py (same names, argument lists and error behaviour,
reference file:line cited per function) over torch tensors, executed by the sm_90a kernels in
libpnp_b200.so.  NHWC activations, HWIO weights, strides as 4-lists [1,s,s,1] -- as in the reference.

Differences a TF-1 user must know:
  * eager, not graph: `is_train` / `keep_prob` are plain Python values at call time;
  * `batch_norm(scope=None)` draws a fresh 'BatchNorm_k' scope on every call (TF build-time
    semantics); pass an explicit scope to re-use statistics across steps (the models do);
  * conv -> dropout -> BN -> activation (+ residual skip) run as ONE fused op per layer.
"""
import torch

from . import functional as F
from . import runtime as rt

def _act_code(leak):
    # the reference tests `leak is True` (layers.py:11,34,163,186): anything else means plain relu
    return F.ACT_LRELU if leak is True else F.ACT_RELU


def _stride_of(strides):
    if len(strides) != 4 or strides[0] != 1 or strides[3] != 1 or strides[1] != strides[2]:
        raise ValueError("strides must be [1, s, s, 1], got %r" % (strides,))
    return int(strides[1])


# ---- variable factories (layers.py:47-62) ---------------------------------------------------------
def _truncated_normal(shape, stddev):
    t = torch.empty(tuple(shape), dtype=torch.float32, device=rt.device())
    torch.nn.init.trunc_normal_(t, mean=0.0, std=stddev, a=-2 * stddev, b=2 * stddev)
    return t


def weight_variable(shape, stddev=0.01, trainable=True):
    """layers.py:47-49 -- tf.Variable(tf.truncated_normal(shape, stddev))"""
    t = _truncated_normal(shape, stddev)
    t.requires_grad_(bool(trainable))
    return rt.new_variable(t, trainable)


def sharable_weight_variable(shape, stddev=0.1, trainable=True, name="IhaveNoName"):
    """layers.py:51-55 -- tf.get_variable under the current variable scope (AUTO_REUSE sharing)"""
    def make():
        t = _truncated_normal(shape, stddev)
        t.requires_grad_(bool(trainable))
        return t
    return rt.get_variable(name, make, trainable)


def weight_variable_deconv(shape, stddev=0.1):
    """layers.py:57-58 (dead code in the reference graph; kept for surface completeness)"""
    return weight_variable(shape, stddev=stddev, trainable=True)


def bias_variable(shape):
    """layers.py:60-62 -- constant 0.1"""
    t = torch.full(tuple(shape), 0.1, dtype=torch.float32, device=rt.device())
    t.requires_grad_(True)
    return rt.new_variable(t, True)


# ---- batch norm variables -------------------------------------------------------------------------
def bn_variables(scope, channels, trainable=True):
    """beta/gamma/moving_mean/moving_variance of tf.contrib.layers.batch_norm under `scope`
    (layers.py:100; names as in lists/pred_bn_list).  Re-used if they already exist."""
    if scope is None:
        scope = rt.default_scope_name("BatchNorm")
    dev = rt.device()

    def mk(val, grad):
        def f():
            t = torch.full((channels,), val, dtype=torch.float32, device=dev)
            t.requires_grad_(grad)
            return t
        return f
    import contextlib
    # a leading '/' makes the scope absolute (the source segmenter's anonymous 'BatchNorm_k' scopes are
    # top-level because tf.name_scope does not prefix tf.get_variable names, lists/old_bn_list)
    outer = rt.root_scope() if scope.startswith("/") else contextlib.nullcontext()
    with outer, rt.variable_scope(scope.lstrip("/")):
        beta = rt.get_variable("beta", mk(0.0, bool(trainable)), trainable, "bn_beta")
        gamma = rt.get_variable("gamma", mk(1.0, bool(trainable)), trainable, "bn_gamma")
        mm = rt.get_variable("moving_mean", mk(0.0, False), False, "bn_moving")
        mv = rt.get_variable("moving_variance", mk(1.0, False), False, "bn_moving")
    return F.BNVars(gamma, beta, mm, mv)


# ---- convolution family -----------------------------------------------------------------------------
def conv2d(x, W, keep_prob_, strides=[1, 1, 1, 1], padding='SAME'):
    """layers.py:64-74: dropout(conv(x, W)); padding 'SAME' or 'SYMMETRIC' (mirror pad k//2 + VALID)."""
    cfg = F.LayerCfg(stride=_stride_of(strides), padding=padding, keep_prob=keep_prob_)
    return F.conv_layer(x, W, cfg)


def conv_bn_2d(x, W, keep_prob, padding='SAME', strides=[1, 1, 1, 1], is_train=True, scope=None, bn_trainable=True):
    """layers.py:16-27: conv -> dropout -> batch_norm"""
    bn = bn_variables(scope, W.shape[3], bn_trainable)
    cfg = F.LayerCfg(stride=_stride_of(strides), padding=padding, keep_prob=keep_prob, bn=bn, bn_training=is_train)
    return F.conv_layer(x, W, cfg)


def conv_bn_relu2d(x, W, keep_prob, padding='SAME', strides=[1, 1, 1, 1], is_train=True, scope=None, bn_trainable=True,
                   leak=False):
    """layers.py:9-14"""
    bn = bn_variables(scope, W.shape[3], bn_trainable)
    cfg = F.LayerCfg(stride=_stride_of(strides), padding=padding, keep_prob=keep_prob, bn=bn, bn_training=is_train,
                     act=_act_code(leak))
    return F.conv_layer(x, W, cfg)


def conv_relu2d(x, W, keep_prob, padding='SAME', strides=[1, 1, 1, 1], leak=False):
    """layers.py:77-82"""
    cfg = F.LayerCfg(stride=_stride_of(strides), padding=padding, keep_prob=keep_prob, act=_act_code(leak))
    return F.conv_layer(x, W, cfg)


def dilate_conv2d(x, W, keep_prob_, rate=2, padding='SAME'):
    """layers.py:84-93: tf.nn.atrous_conv2d + dropout"""
    cfg = F.LayerCfg(dil=int(rate), padding=padding, keep_prob=keep_prob_)
    return F.conv_layer(x, W, cfg)


def dilate_conv_bn(x, W, keep_prob, padding='SAME', rate=2, is_train=True, scope=None, bn_trainable=True):
    """layers.py:39-45"""
    bn = bn_variables(scope, W.shape[3], bn_trainable)
    cfg = F.LayerCfg(dil=int(rate), padding=padding, keep_prob=keep_prob, bn=bn, bn_training=is_train)
    return F.conv_layer(x, W, cfg)


def dilate_conv_bn_relu2d(x, W, keep_prob, padding='SAME', rate=2, is_train=True, scope=None, bn_trainable=True, leak=False):
    """layers.py:29-37"""
    bn = bn_variables(scope, W.shape[3], bn_trainable)
    cfg = F.LayerCfg(dil=int(rate), padding=padding, keep_prob=keep_prob, bn=bn, bn_training=is_train, act=_act_code(leak))
    return F.conv_layer(x, W, cfg)


def batch_norm(x, is_training=True, scope=None, trainable=True):
    """layers.py:95-100 as a standalone op (identity 1x1 structure is not needed: BN-only apply)."""
    C = x.shape[-1]
    bn = bn_variables(scope, C, trainable)
    return _BNOnly.apply(x, bn, bool(is_training), bn.gamma, bn.beta)


class _BNOnly(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bn, training, gamma, beta):
        from ._C import call, ptr
        x = x.contiguous()
        C = x.shape[-1]
        M = x.numel() // C
        dev = x.device
        stats = F._zeros_f64(2 * C, dev) if training else None
        if training:
            call("pnp_bn_stats", ptr(x), M, C, ptr(stats[:C]), ptr(stats[C:]), rt.stream())
        vec = torch.empty(4, C, dtype=torch.float32, device=dev)
        call("pnp_bn_finalize", ptr(stats[:C]) if training else None, ptr(stats[C:]) if training else None, M, C, ptr(bn.gamma),
             ptr(bn.beta), ptr(bn.moving_mean), ptr(bn.moving_var), 1 if training else 0, ptr(vec[0]), ptr(vec[1]), ptr(vec[2]),
             ptr(vec[3]), rt.stream())
        if training:
            bn.moving_mean.pnp_version = getattr(bn.moving_mean, "pnp_version", 0) + 1
            bn.moving_var.pnp_version = getattr(bn.moving_var, "pnp_version", 0) + 1
        y = torch.empty_like(x)
        call("pnp_bn_act_apply", ptr(x), ptr(vec[0]), ptr(vec[1]), None, 0, 0, F.ACT_NONE, ptr(y), None, None, M, C, rt.stream())
        ctx.save_for_backward(x)
        ctx.meta = (bn, training, vec, M, C)
        return y

    @staticmethod
    def backward(ctx, dy):
        from ._C import call, ptr
        (x,) = ctx.saved_tensors
        bn, training, vec, M, C = ctx.meta
        dy = dy.contiguous()
        dev = dy.device
        g = torch.empty_like(dy)
        sums = F._zeros_f64(2 * C, dev)
        call("pnp_bn_bwd_reduce", ptr(dy), None, ptr(x), ptr(vec[2]), ptr(vec[3]), F.ACT_NONE, ptr(g), ptr(sums[:C]), ptr(sums[C:]),
             M, C, rt.stream())
        coef = torch.empty(2 * C, dtype=torch.float32, device=dev)
        dgamma = F._grad_slot(bn.gamma) if bn.gamma.requires_grad else None
        dbeta = F._grad_slot(bn.beta) if bn.beta.requires_grad else None
        call("pnp_bn_bwd_finalize", ptr(sums[:C]), ptr(sums[C:]), M, C, ptr(dgamma), ptr(dbeta), ptr(coef), rt.stream())
        dx = torch.empty_like(dy)
        call("pnp_bn_bwd_apply", ptr(g), ptr(x), ptr(vec[2]), ptr(vec[3]), ptr(bn.gamma), ptr(coef), 1 if training else 0, None,
             ptr(dx), None, None, M, C, rt.stream())
        return dx, None, None, None, None


# ---- pooling / concat / softmax ------------------------------------------------------------------------
def max_pool2d(x, n):
    """layers.py:102-103: tf.nn.max_pool, ksize = strides = [1,n,n,1], 'SAME'.  n = 2 on even maps (every use in the reference
    graphs) takes the vectorised 2x2 kernel; any other n / odd maps the general SAME-geometry kernel."""
    n = int(n)
    if n < 1:
        raise ValueError("max_pool2d: n must be a positive integer")
    if n == 2 and x.shape[1] % 2 == 0 and x.shape[2] % 2 == 0:
        return F.max_pool2(x)
    return F.pool_same(x, n, avg=False)


def avg_pool2d(x, n):
    """layers.py:105-106: tf.nn.avg_pool, ksize = strides = [1,n,n,1], 'SAME' (padding is not counted).  Never called by the reference
    graphs."""
    n = int(n)
    if n < 1:
        raise ValueError("avg_pool2d: n must be a positive integer")
    if n == 2 and x.shape[1] % 2 == 0 and x.shape[2] % 2 == 0:
        return F.avg_pool2(x)
    return F.pool_same(x, n, avg=True)


def simple_concat2d(x1, x2):
    """layers.py:117-127: channel concat; the reference's shape check is a no-op, ours raises the same
    ValueError when the leading dims differ.  (The discriminator input uses the fused gather instead.)"""
    if tuple(x1.shape[:-1]) != tuple(x2.shape[:-1]):
        print("x1_shape: %s" % str(list(x1.shape)))
        print("x2_shape: %s" % str(list(x2.shape)))
        raise ValueError("Cannot concatenate tensors with different shape, igonoring feature map depth")
    return F.crop_concat(x1, x2)


def crop_and_concat(x1, x2, name="default"):
    """layers.py:108-115 -- centre-crop x1 to x2's height and width (offsets (H1-H2)//2, (W1-W2)//2) and concat along channels
    (unused by the reference graphs)"""
    if x1.shape[0] != x2.shape[0] or x1.shape[1] < x2.shape[1] or x1.shape[2] < x2.shape[2]:
        raise ValueError("crop_and_concat: x1 %s cannot be cropped to x2 %s" % (list(x1.shape), list(x2.shape)))
    return F.crop_concat(x1, x2)


def pixel_wise_softmax_2(output_map):
    """layers.py:134-138: exp/sum over channels without max subtraction, clipped to +-1e15"""
    return F.pixel_softmax2(output_map)


def pixel_wise_softmax(output_map):
    """layers.py:129-132: two-class special case e/(e + reverse(e)) == softmax over 2 channels"""
    if output_map.shape[-1] != 2:
        raise ValueError("pixel_wise_softmax is the 2-class form; use pixel_wise_softmax_2")
    return F.pixel_softmax2(output_map)


def cross_entropy(y_, output_map):
    """layers.py:140-141: -mean(y_ * log(clip(output_map, 1e-10, 1))) (unused by the reference graphs)"""
    if tuple(y_.shape) != tuple(output_map.shape):
        raise ValueError("cross_entropy: labels %s and probabilities %s differ in shape" % (list(y_.shape), list(output_map.shape)))
    return F.cross_entropy(y_, output_map)


# ---- residual blocks -----------------------------------------------------------------------------------
def _block(x, w1, w2, keep_prob, inc_dim, is_train, scope, bn_trainable, leak, padding, dil):
    s1 = None if scope is None else scope + "_1"
    s2 = None if scope is None else scope + "_2"
    cin = x.shape[-1]
    bn1 = bn_variables(s1, w1.shape[3], bn_trainable)
    bn2 = bn_variables(s2, w2.shape[3], bn_trainable)
    act = _act_code(leak)
    cfg1 = F.LayerCfg(dil=dil, padding=padding, keep_prob=keep_prob, bn=bn1, bn_training=is_train, act=act)
    # x_s = x zero-padded by cin//2 channels on both sides when inc_dim (layers.py:160,182)
    cfg2 = F.LayerCfg(dil=dil, padding=padding, keep_prob=keep_prob, bn=bn2, bn_training=is_train, act=act,
                      skip_off=(cin // 2 if inc_dim is True else 0))
    if inc_dim is not True and w2.shape[3] != cin:
        raise ValueError("residual add: %d vs %d channels (set inc_dim=True?)" % (cin, w2.shape[3]))
    return F.res_block(x, w1, w2, cfg1, cfg2)


def residual_block(x, w1, w2, keep_prob, inc_dim=False, is_train=True, scope=None, bn_trainable=True, leak=False,
                   padding='SAME'):
    """layers.py:145-166"""
    return _block(x, w1, w2, keep_prob, inc_dim, is_train, scope, bn_trainable, leak, padding, 1)


def DR_block(x, w1, w2, rate, keep_prob, inc_dim=False, is_train=True, bn_trainable=True, scope=None, leak=False):
    """layers.py:168-189"""
    return _block(x, w1, w2, keep_prob, inc_dim, is_train, scope, bn_trainable, leak, 'SAME', int(rate))
