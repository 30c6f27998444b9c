"""numpy float32 restatement of what the reference's image summaries compute, for the image-summary tests.

* `image_summary_u8`: TF-1.4 ImageSummaryOp on a float [B, H, W, 1] tensor (summary_image_op.cc, NormalizeFloatImage): images
  0..min(B, max_outputs)-1, each normalised on its own -- min / max over the finite pixels; a negative min maps 0 to 128 with
  scale 127 / max(|min|, |max|), otherwise [0, max] maps to [0, 255] with scale 255 / max; scale 0 below 1e-6; pixel =
  uint8(trunc(v * scale + offset)) with the product and the sum each rounded to float32; non-finite pixels take bad_color[0] = 255.
* `first_argmax`: tf.argmax over the last axis (first maximal index), `pixel_softmax2`: layers.py:134-138 (no max subtraction,
  the +-1e15 clip), both in float32.
"""
import numpy as np


def image_summary_u8(nhwc_float32, max_outputs=3):
    x = np.asarray(nhwc_float32)
    assert x.dtype == np.float32 and x.ndim == 4 and x.shape[3] == 1, (x.dtype, x.shape)
    n = min(x.shape[0], int(max_outputs))
    out = np.empty((n,) + x.shape[1:3], np.uint8)
    for i in range(n):
        v = x[i, :, :, 0]
        fin = np.isfinite(v)
        mn = v[fin].min() if fin.any() else np.float32(np.inf)
        mx = v[fin].max() if fin.any() else np.float32(-np.inf)
        if mn < 0:
            max_val = np.maximum(np.abs(mn), np.abs(mx))
            scale = np.float32(0) if max_val < np.float32(1e-6) else np.float32(127) / max_val
            offset = np.float32(128)
        else:
            scale = np.float32(0) if mx < np.float32(1e-6) else np.float32(255) / mx
            offset = np.float32(0)
        vf = np.where(fin, v, np.float32(0))
        y = (vf * np.float32(scale)).astype(np.float32) + np.float32(offset)
        assert y.dtype == np.float32
        out[i] = np.where(fin, np.trunc(y), np.float32(255)).astype(np.uint8)
    return out


def first_argmax(x):
    """index of the first maximum along the last axis, as tf.argmax returns it, with a strict '>' scan"""
    x = np.asarray(x, np.float32)
    best = x[..., 0].copy()
    arg = np.zeros(x.shape[:-1], np.int64)
    for c in range(1, x.shape[-1]):
        m = x[..., c] > best
        best = np.where(m, x[..., c], best)
        arg = np.where(m, c, arg)
    return arg


def pixel_softmax2(logits):
    e = np.exp(np.asarray(logits, np.float32))
    s = np.zeros(e.shape[:-1], np.float32)
    for c in range(e.shape[-1]):
        s = s + e[..., c]
    return np.clip(e / s[..., None], np.float32(-1e15), np.float32(1e15)).astype(np.float32)


def compact_panels(arg_map, max_outputs=3):
    """image_summary_u8 of tf.expand_dims(tf.cast(arg_map, tf.float32), 3)"""
    return image_summary_u8(np.asarray(arg_map).astype(np.float32)[..., None], max_outputs)
