"""
ORACLE (test infrastructure, NOT product code) -- torch-CPU restatement of the reference's
layers.py / ops.py operator surface with TensorFlow-1.4 semantics, differentiable through torch
autograd so that backward passes and optimizer steps can be checked too.

PARITY UNPINNED for the TF-kernel numerics (see oracle/tf14_numpy.py header): no reference tests / golden vectors exist
and TF-1.4 cannot run here; this form is cross-checked against the naive numpy form and hand-derived known-answer
tests.  PS, softmax_weighted_loss and dice_loss ARE pinned to the reference's own code executed in this container
(tests/test_reference_golden.py, tests/test_reference_graph_trace.py).

Tensors are NHWC at the interface (like the reference) and permuted to NCHW internally for
torch.nn.functional.conv2d.  Weights are HWIO.  dtype follows the inputs (fp32 for timing /
CPU baseline, fp64 for tight parity checks).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this.
"""
import math
import torch
import torch.nn.functional as F

from .tf14_numpy import same_pad, BN_DECAY, BN_EPS


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def symmetric_pad(x, p):
    """tf.pad(x, [[0,0],[p,p],[p,p],[0,0]], 'SYMMETRIC') on NHWC (layers.py:19-23): mirror that
    includes the edge element.  torch has no 'symmetric' mode, so build it from flips."""
    if p == 0:
        return x
    top = x[:, :p].flip(1)
    bot = x[:, -p:].flip(1)
    x = torch.cat([top, x, bot], dim=1)
    left = x[:, :, :p].flip(2)
    right = x[:, :, -p:].flip(2)
    return torch.cat([left, x, right], dim=2)


def conv2d_raw(x, w, stride=1, dilation=1, padding="SAME"):
    """tf.nn.conv2d / atrous_conv2d (layers.py:18-24,67-73,86-92) without dropout."""
    kh, kw = w.shape[0], w.shape[1]
    if padding == "SYMMETRIC":
        x = symmetric_pad(x, kh // 2)
        padding = "VALID"
    H, W = x.shape[1], x.shape[2]
    xn = _nchw(x)
    if padding == "SAME":
        pt, pb = same_pad(H, kh, stride, dilation)
        pl, pr = same_pad(W, kw, stride, dilation)
        xn = F.pad(xn, (pl, pr, pt, pb))
    wn = w.permute(3, 2, 0, 1)  # HWIO -> OIHW
    y = F.conv2d(xn, wn, stride=stride, dilation=dilation)
    return _nhwc(y)


def dropout(x, keep_prob, mask=None):
    """tf.nn.dropout (layers.py:25,74,93): x * floor(keep + U) / keep, U from torch's generator here.  Parity runs use
    keep_prob == 1 (identity), an injected 0/1 mask, or replace this function by tests/models.PhiloxMasks, which applies the
    library's own Philox masks (tests/test_dropout_model_gpu.py)."""
    if mask is not None:
        return x * mask / keep_prob
    if keep_prob >= 1.0:
        return x
    m = torch.floor(keep_prob + torch.rand_like(x))
    return x * m / keep_prob


class BNState:
    """beta/gamma/moving_mean/moving_variance of one tf.contrib.layers.batch_norm scope."""

    def __init__(self, C, dtype=torch.float32):
        self.gamma = torch.ones(C, dtype=dtype, requires_grad=True)
        self.beta = torch.zeros(C, dtype=dtype, requires_grad=True)
        self.moving_mean = torch.zeros(C, dtype=dtype)
        self.moving_var = torch.ones(C, dtype=dtype)


def batch_norm(x, bn, is_training):
    """layers.py:95-100 (see tf14_numpy.batch_norm).  Mutates bn.moving_* when training."""
    C = x.shape[-1]
    if is_training:
        flat = x.reshape(-1, C)
        n = flat.shape[0]
        mean = flat.mean(0)
        var = ((flat - mean) ** 2).mean(0)
        y = (x - mean) * torch.rsqrt(var + BN_EPS) * bn.gamma + bn.beta
        with torch.no_grad():
            unbiased = var * (n / max(n - 1, 1))
            bn.moving_mean = BN_DECAY * bn.moving_mean + (1 - BN_DECAY) * mean.detach()
            bn.moving_var = BN_DECAY * bn.moving_var + (1 - BN_DECAY) * unbiased.detach()
        return y
    return (x - bn.moving_mean) * torch.rsqrt(bn.moving_var + BN_EPS) * bn.gamma + bn.beta


def act(x, leak):
    """tf.nn.leaky_relu (alpha 0.2) if leak else tf.nn.relu (layers.py:11-14)."""
    return F.leaky_relu(x, 0.2) if leak else F.relu(x)


def conv2d(x, W, keep_prob_, strides=(1, 1, 1, 1), padding="SAME"):
    """layers.py:64-74."""
    return dropout(conv2d_raw(x, W, stride=strides[1], padding=padding), keep_prob_)


def conv_bn_2d(x, W, keep_prob, bn, padding="SAME", strides=(1, 1, 1, 1), is_train=True):
    """layers.py:16-27: conv -> dropout -> BN."""
    return batch_norm(dropout(conv2d_raw(x, W, stride=strides[1], padding=padding), keep_prob), bn, is_train)


def conv_bn_relu2d(x, W, keep_prob, bn, padding="SAME", strides=(1, 1, 1, 1), is_train=True, leak=False):
    """layers.py:9-14."""
    return act(conv_bn_2d(x, W, keep_prob, bn, padding, strides, is_train), leak)


def dilate_conv2d(x, W, keep_prob_, rate=2, padding="SAME"):
    """layers.py:84-93."""
    return dropout(conv2d_raw(x, W, dilation=rate, padding=padding), keep_prob_)


def dilate_conv_bn(x, W, keep_prob, bn, rate=2, is_train=True):
    """layers.py:39-45."""
    return batch_norm(dilate_conv2d(x, W, keep_prob, rate), bn, is_train)


def channel_pad_skip(x):
    """layers.py:160,182."""
    C = x.shape[-1]
    return F.pad(x, (C // 2, C // 2))


def residual_block(x, w1, w2, keep_prob, bn1, bn2, inc_dim=False, is_train=True, leak=False, padding="SAME"):
    """layers.py:145-166."""
    h = conv_bn_relu2d(x, w1, keep_prob, bn1, padding=padding, is_train=is_train, leak=leak)
    h = conv_bn_2d(h, w2, keep_prob, bn2, padding=padding, is_train=is_train)
    xs = channel_pad_skip(x) if inc_dim else x
    return act(xs + h, leak)


def DR_block(x, w1, w2, rate, keep_prob, bn1, bn2, inc_dim=False, is_train=True, leak=False):
    """layers.py:168-189."""
    h = act(dilate_conv_bn(x, w1, keep_prob, bn1, rate, is_train), leak)
    h = dilate_conv_bn(h, w2, keep_prob, bn2, rate, is_train)
    xs = channel_pad_skip(x) if inc_dim else x
    return act(xs + h, leak)


def max_pool2d(x, n=2):
    """layers.py:102-103 (even dims => SAME == VALID)."""
    return _nhwc(F.max_pool2d(_nchw(x), n, n))


def pool_same(x, n, avg=False):
    """layers.py:102-106 for any n and any map size: TF 'SAME' geometry (tf14_numpy.pool_same), differentiable"""
    B, H, W, C = x.shape
    Ho, Wo = -(-H // n), -(-W // n)
    pt, pl = (Ho * n - H) // 2, (Wo * n - W) // 2
    pad = (pl, Wo * n - W - pl, pt, Ho * n - H - pt)
    xc = _nchw(x)
    if not avg:
        return _nhwc(F.max_pool2d(F.pad(xc, pad, value=float("-inf")), n, n))
    ssum = F.avg_pool2d(F.pad(xc, pad), n, n) * (n * n)
    cnt = F.avg_pool2d(F.pad(torch.ones(1, 1, H, W, dtype=x.dtype), pad), n, n) * (n * n)
    return _nhwc(ssum / cnt)


def crop_and_concat(x1, x2):
    """layers.py:108-115"""
    oy, ox = (x1.shape[1] - x2.shape[1]) // 2, (x1.shape[2] - x2.shape[2]) // 2
    return torch.cat([x1[:, oy:oy + x2.shape[1], ox:ox + x2.shape[2], :], x2], 3)


def cross_entropy(y_, output_map):
    """layers.py:140-141; torch.clamp passes the gradient inside [min, max] (bounds included) like tf.clip_by_value"""
    return -torch.mean(y_ * torch.log(torch.clamp(output_map, 1e-10, 1.0)))


def PS(X, r, n_channel, batch_size):
    """ops.py:23-27 via the closed-form index law pinned in tests/test_oracle_kat.py against the
    literal emulation (tf14_numpy.PS_literal).
       B>=2: out[n, i*r+q, j*r+p, g] = X[n, i, j, g*r*r + p*r + q]   (p = column offset)
       B==1: out[n, i*r+p, j*r+q, g] = X[n, i, j, g*r*r + p*r + q]"""
    B, a, b, C = X.shape
    assert B == batch_size and C == n_channel * r * r
    Xv = X.reshape(B, a, b, n_channel, r, r)  # [..., g, p, q]
    if B >= 2:
        out = Xv.permute(0, 1, 5, 2, 4, 3)  # B, i, q, j, p, g
    else:
        out = Xv.permute(0, 1, 4, 2, 5, 3)  # B, i, p, j, q, g
    return out.reshape(B, a * r, b * r, n_channel)


def pixel_wise_softmax_2(x):
    """layers.py:134-138."""
    e = torch.exp(x)
    return torch.clamp(e / e.sum(3, keepdim=True), -1e15, 1e15)


def softmax_weighted_loss(logits, y):
    """source_segmenter.py:241-258."""
    p = torch.softmax(logits, dim=-1)
    tot = y.sum()
    raw = 0
    for i in range(y.shape[-1]):
        gti = y[..., i]
        wi = 1 - gti.sum() / tot
        raw = raw + -1.0 * wi * gti * torch.log(torch.clamp(p[..., i], 0.005, 1))
    return raw.mean()


def dice_loss(logits, y):
    """source_segmenter.py:260-273."""
    p = torch.softmax(logits, dim=-1)
    dice = 0
    for i in range(y.shape[-1]):
        inse = (p[..., i] * y[..., i]).sum()
        l = (p[..., i] * p[..., i]).sum()
        r = y[..., i].sum()
        dice = dice + 2.0 * inse / (l + r + 1e-7)
    return -1.0 * dice / y.shape[-1]


def dice_eval(compact_pred, labels, n_class):
    """lib.py:96-110."""
    pred = F.one_hot(compact_pred, n_class).to(labels.dtype)
    arr = []
    for i in range(n_class):
        inse = (pred[..., i] * labels[..., i]).sum()
        union = pred[..., i].sum() + labels[..., i].sum()
        arr.append(2.0 * inse / (union + 1e-7))
    return sum(arr) / n_class, arr


def l2_loss(w):
    """tf.nn.l2_loss."""
    return (w * w).sum() / 2


class TFAdam:
    """tf.train.AdamOptimizer (source_segmenter.py:378), TF defaults."""

    def __init__(self, params, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8):
        self.params = list(params)
        self.lr, self.b1, self.b2, self.eps = lr, b1, b2, eps
        self.m = [torch.zeros_like(p) for p in self.params]
        self.v = [torch.zeros_like(p) for p in self.params]
        self.t = 0

    @torch.no_grad()
    def step(self, grads):
        self.t += 1
        lr_t = self.lr * math.sqrt(1 - self.b2 ** self.t) / (1 - self.b1 ** self.t)
        for p, g, m, v in zip(self.params, grads, self.m, self.v):
            if g is None:
                continue
            m.mul_(self.b1).add_(g, alpha=1 - self.b1)
            v.mul_(self.b2).addcmul_(g, g, value=1 - self.b2)
            p.sub_(lr_t * m / (v.sqrt() + self.eps))


class TFRMSProp:
    """tf.train.RMSPropOptimizer (adversarial.py:643-652): decay .9, momentum 0, eps 1e-10 inside the
    sqrt, ms initialised to ONE."""

    def __init__(self, params, lr=3e-4, decay=0.9, momentum=0.0, eps=1e-10):
        self.params = list(params)
        self.lr, self.decay, self.momentum, self.eps = lr, decay, momentum, eps
        self.ms = [torch.ones_like(p) for p in self.params]
        self.mom = [torch.zeros_like(p) for p in self.params]

    @torch.no_grad()
    def step(self, grads):
        for p, g, ms, mom in zip(self.params, grads, self.ms, self.mom):
            if g is None:
                continue
            ms.mul_(self.decay).addcmul_(g, g, value=1 - self.decay)
            mom.mul_(self.momentum).add_(self.lr * g / torch.sqrt(ms + self.eps))
            p.sub_(mom)
