"""ctypes binding of the C-ABI in include/pnp_b200.h (libpnp_b200.so, built in-tree by _build.py).

There is no CPU fallback: if the library is missing the import raises, and every launcher raises
RuntimeError on a non-zero return code."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpnp_b200.so")

c_void_p, c_int, c_ll, c_float, c_ull = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_ulonglong


class ConvGeom(ctypes.Structure):
    """pnp_conv_geom"""
    _fields_ = [(n, c_int) for n in ("B", "H", "W", "Cin", "Ho", "Wo", "Cout", "kh", "kw", "stride", "dil", "pad_t", "pad_l")]


class DropCfg(ctypes.Structure):
    """pnp_dropout_cfg"""
    _fields_ = [("seed_ptr", c_void_p), ("stream", c_ull), ("keep", c_float)]


class TcEpilogue(ctypes.Structure):
    """pnp_tc_epilogue"""
    _fields_ = [("scale", c_void_p), ("shift", c_void_p), ("skip", c_void_p), ("skip_C", c_int), ("skip_off", c_int), ("act", c_int),
                ("y_hi", c_void_p), ("y_lo", c_void_p)]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "libpnp_b200.so not found at %s -- run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU/PyTorch fallback for the CUDA hot path)" % LIB_PATH)
    return ctypes.CDLL(LIB_PATH)


lib = _load()

P = c_void_p
_GEOM = ctypes.POINTER(ConvGeom)
_DROP = ctypes.POINTER(DropCfg)

# name -> argtypes, mirrors include/pnp_b200.h one to one
SIGNATURES = {
    "pnp_conv2d_fwd": [P, P, P, _GEOM, _DROP, c_int, P],
    "pnp_conv2d_dgrad": [P, P, P, _GEOM, c_int, P],
    "pnp_conv2d_wgrad": [P, P, P, _GEOM, P],
    "pnp_weight_transpose": [P, P, c_int, c_int, c_int, P],
    "pnp_ps_mirror_conv_fwd": [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_ps_mirror_conv_bwd": [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_split_bf16": [P, P, P, c_ll, P],
    "pnp_split_weight_bf16": [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_split_bf16_pad": [P, P, P, c_ll, c_int, c_int, P],
    "pnp_conv2d_tc_fwd": [P, P, P, P, P, _GEOM, c_int, _DROP, c_int, P, P, P],
    "pnp_conv2d_tc_fwd_fused": [P, P, P, P, P, _GEOM, c_int, _DROP, c_int, P, P, ctypes.POINTER(TcEpilogue), P],
    "pnp_conv2d_tc_dgrad": [P, P, P, P, P, _GEOM, c_int, c_int, P],
    "pnp_conv2d_tc_wgrad": [P, P, P, P, P, _GEOM, c_int, c_int, P],
    "pnp_bn_stats": [P, c_ll, c_int, P, P, P],
    "pnp_bn_finalize": [P, P, c_ll, c_int, P, P, P, P, c_int, P, P, P, P, P],
    "pnp_bn_act_apply": [P, P, P, P, c_int, c_int, c_int, P, P, P, c_ll, c_int, P],
    "pnp_bn_apply_fused": [P, P, P, c_ll, c_int, P, P, P, P, c_int, P, c_int, c_int, c_int, P, P, P, P, P, P],
    "pnp_bn_bwd_apply_fused": [P, P, P, P, P, P, P, c_ll, c_int, c_int, _DROP, P, P, P, P, P, P],
    "pnp_bn_bwd_reduce_sums": [P, P, P, P, P, P, c_int, P, P, c_ll, c_int, P],
    "pnp_bn_bwd_apply_direct": [P, P, P, c_int, P, P, P, P, P, P, c_ll, c_int, c_int, _DROP, P, P, P, P, P, P],
    "pnp_bn_bwd_reduce": [P, P, P, P, P, c_int, P, P, P, c_ll, c_int, P],
    "pnp_bn_bwd_finalize": [P, P, c_ll, c_int, P, P, P, P],
    "pnp_bn_bwd_apply": [P, P, P, P, P, P, c_int, _DROP, P, P, P, c_ll, c_int, P],
    "pnp_act_bwd": [P, P, c_int, P, c_ll, P],
    "pnp_channel_slice": [P, c_int, c_int, c_int, P, c_ll, c_int, P],
    "pnp_dropout_apply": [P, P, c_ll, _DROP, P],
    "pnp_seed_advance": [P, P],
    "pnp_maxpool2_fwd": [P, P, c_int, c_int, c_int, c_int, P],
    "pnp_maxpool2_bwd": [P, P, P, c_int, c_int, c_int, c_int, P],
    "pnp_avgpool2": [P, P, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_pool_fwd": [P, P, c_int, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_pool_bwd": [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_crop_concat_fwd": [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_crop_concat_bwd": [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_cross_entropy_fwd": [P, P, c_ll, P, P, P],
    "pnp_cross_entropy_bwd": [P, P, P, c_ll, P, P, P],
    "pnp_mirror_pad_fwd": [P, P, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_mirror_pad_bwd": [P, P, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_phase_shift_fwd": [P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_phase_shift_bwd": [P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_logits_argmax_concat": [P, P, c_ll, c_int, c_int, c_int, P],
    "pnp_disc_input_fwd": [P, P, P, P, P, c_int, P, c_int, P, c_int, c_int, c_int, c_int, c_int, P],
    "pnp_pixel_softmax2": [P, P, c_ll, c_int, P],
    "pnp_image_summary_u8": [P, P, P, P, c_int, c_int, c_int, c_int, c_int, P, P],
    "pnp_segloss_reduce": [P, P, c_ll, c_int, P, P],
    "pnp_segloss_finalize": [P, c_ll, c_int, P, P, P],
    "pnp_segloss_bwd": [P, P, P, P, P, P, c_ll, c_int, P],
    "pnp_confusion": [P, P, c_ll, c_int, P, P],
    "pnp_one_hot": [P, P, c_ll, c_int, P],
    "pnp_fc_fwd": [P, P, P, c_int, c_int, P],
    "pnp_fc_bwd": [P, P, P, P, P, c_int, c_int, P],
    "pnp_mean_combo": [P, c_float, P, c_float, c_int, P, P],
    "pnp_l2_loss_acc": [P, c_ll, P, P],
    "pnp_adam_advance": [P, c_float, c_float, P],
    "pnp_adam_step": [P, P, P, P, c_ll, P, P, P, c_float, c_float, c_float, c_float, P],
    "pnp_rmsprop_step": [P, P, P, P, c_ll, P, P, P, P, c_float, c_float, c_float, c_float, P],
    "pnp_momentum_step": [P, P, P, c_ll, P, P, P, c_float, c_float, P],
    "pnp_fill": [P, c_float, c_ll, P],
}

for _name, _args in SIGNATURES.items():
    _f = getattr(lib, _name)
    _f.argtypes = _args
    _f.restype = c_int
lib.pnp_error_string.argtypes = [c_int]
lib.pnp_error_string.restype = ctypes.c_char_p
lib.pnp_version.restype = c_int
lib.pnp_tc_available.restype = c_int
lib.pnp_tc_last_config.argtypes = [P, P, P]
lib.pnp_tc_last_config.restype = c_int

# launch counter: bench.py reports how many of OUR kernels ran inside the timed region
launch_count = 0


ERR_UNSUPPORTED = 100002


class Unsupported(RuntimeError):
    """the launcher declined this shape (PNP_ERR_UNSUPPORTED): callers pick the general kernel instead"""


def call(name, *args):
    global launch_count
    rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = "%s failed: [%d] %s" % (name, rc, lib.pnp_error_string(rc).decode())
        if rc == ERR_UNSUPPORTED:
            raise Unsupported(msg)
        raise RuntimeError(msg)
    launch_count += 1


def ptr(t):
    """device pointer of a torch tensor (None -> NULL)"""
    return None if t is None else t.data_ptr()
