"""ctypes binding of the C-ABI shared library ``libseg_b200.so`` (declared in ``include/seg_b200.h``).

Every function takes plain device pointers / sizes and a ``cudaStream_t``; torch is used only to own device memory
and streams.  There is no CPU fallback: if the library is missing or the device is not sm_90 the import-time /
first-call checks raise.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_uint8, c_uint32, c_uint64, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libseg_b200.so")

DT_BF16, DT_F32 = 0, 1
IMPL_AUTO, IMPL_SIMT, IMPL_TC = 0, 1, 2
LOSS_CE, LOSS_WCE, LOSS_FOCAL = 0, 1, 2  # SEG_LOSS_* (the `kind` of the seg_loss_* / seg_upsample_loss_* entry points)


class SyncDesc(Structure):
    """Mirror of ``seg_sync_desc`` (include/seg_b200.h)."""

    _fields_ = [("peers", c_void_p), ("rank", c_int32), ("world", c_int32), ("n_max", c_int32), ("timeout_clocks", c_int64)]


class ConvDesc(Structure):
    """Mirror of ``seg_conv_desc`` (include/seg_b200.h)."""

    _fields_ = [(n, c_int32) for n in ("N", "H", "W", "C", "K", "R", "S", "stride", "pad", "dil", "P", "Q", "ldx", "ldy")]


def conv_out_size(size, k, stride, pad, dil):
    return (size + 2 * pad - dil * (k - 1) - 1) // stride + 1


def make_conv_desc(N, H, W, C, K, R, S, stride, pad, dil, ldx=None, ldy=None):
    P = conv_out_size(H, R, stride, pad, dil)
    Q = conv_out_size(W, S, stride, pad, dil)
    return ConvDesc(N, H, W, C, K, R, S, stride, pad, dil, P, Q, ldx if ldx is not None else C, ldy if ldy is not None else K)


_SIGS = {
    "seg_last_error": (c_char_p, []),
    "seg_version": (c_int, []),
    "seg_device_ok": (c_int, []),
    "seg_launch_count": (c_int64, []),
    "seg_launch_count_reset": (None, []),
    "seg_conv2d_fwd": (c_int, [POINTER(ConvDesc), c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "seg_conv2d_dgrad": (c_int, [POINTER(ConvDesc), c_void_p, c_void_p, c_void_p, c_float, c_int, c_void_p]),
    "seg_conv2d_wgrad_workspace_floats": (c_int64, [POINTER(ConvDesc), c_int]),
    "seg_conv2d_wgrad": (c_int, [POINTER(ConvDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "seg_dwconv_scratch_floats": (c_int64, [c_int]),
    "seg_dwconv3x3_fwd": (c_int, [POINTER(ConvDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "seg_dwconv3x3_bwd_data": (c_int, [POINTER(ConvDesc), c_void_p, c_void_p, c_void_p, c_float, c_void_p]),
    "seg_dwconv3x3_bwd_weight": (c_int, [POINTER(ConvDesc), c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p]),
    "seg_dw_pack_weight": (c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    "seg_dw_unpack_wgrad": (c_int, [c_void_p, c_void_p, c_int, c_float, c_void_p]),
    "seg_pack_weight": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_unpack_wgrad": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "seg_pack_entry_bytes": (c_int, []),
    "seg_pack_weights_batched": (c_int, [c_void_p, c_int, c_int64, c_void_p]),
    "seg_unpack_wgrads_batched": (c_int, [c_void_p, c_int, c_int64, c_float, c_void_p]),
    "seg_im2col": (c_int, [POINTER(ConvDesc), c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "seg_bn_stats": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "seg_bn_finalize": (c_int, [c_void_p, c_double, c_int, c_void_p, c_void_p, c_float, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "seg_bn_eval_scale_shift": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p]),
    "seg_bn_apply": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int64, c_int, c_int, c_float, c_uint64, c_void_p, c_int, c_void_p]),
    "seg_counter_add": (c_int, [c_void_p, c_uint64, c_void_p]),
    "seg_bn_bwd_reduce_slots": (c_int, []),
    "seg_bn_bwd_reduce": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int64, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "seg_bn_apply_train": (c_int, [c_void_p, c_int, c_void_p, c_double, c_void_p, c_void_p, c_float, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int64, c_int, c_int, c_float, c_uint64, c_void_p, c_int, c_int, c_int, c_void_p]),
    "seg_bn_bwd_fused_workspace": (c_int, [c_int64, c_int, POINTER(c_int64), POINTER(c_int64)]),
    "seg_bn_bwd_fused": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_double, c_int64, c_int, c_int, c_float,
                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_float, c_int, c_void_p, c_float, c_void_p]),
    "seg_bn_bwd_apply": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_double, c_int64, c_int, c_int, c_float, c_void_p, c_int, c_void_p, c_int, c_float, c_void_p, c_float, c_void_p]),
    "seg_bn_param_grad": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "seg_maxpool3x3s2_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_maxpool3x3s2_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_maxpool2x2_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_maxpool2x2_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_maxunpool2x2_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_maxunpool2x2_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_relu_maxpool2x2_ceil_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_relu_maxpool2x2_ceil_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_avgpool2x2_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_avgpool2x2_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "seg_adaptive_avgpool_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_adaptive_avgpool_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "seg_bilinear_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_bilinear_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "seg_bilinear_logits_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_bilinear_logits_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_pixel_shuffle_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_pixel_shuffle_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "seg_pixel_shuffle_logits_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_pixel_shuffle_logits_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_shuffle_loss_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int64, c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "seg_shuffle_loss_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int64, c_void_p, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "seg_nhwc_loss_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int64, c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "seg_nhwc_loss_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int64, c_void_p, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "seg_dice_nchw_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "seg_dice_nchw_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_float, c_void_p, c_void_p, c_float, c_void_p]),
    "seg_lovasz_count": (c_int, [c_void_p, c_int64, c_int, c_int64, c_void_p, c_void_p]),
    "seg_lovasz_workspace_bytes": (c_int64, [c_int64, c_int, c_int]),
    "seg_lovasz_softmax_nchw": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int64, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "seg_eval_metrics_nchw": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "seg_loss_nchw_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int64, c_void_p, c_int, c_float, c_void_p, c_void_p]),
    "seg_loss_nchw_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int64, c_void_p, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "seg_loss_finalize": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "seg_upsample_loss_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int64, c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "seg_upsample_loss_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int64, c_void_p, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "seg_relu_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int64, c_int, c_void_p]),
    "seg_relu_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int64, c_int, c_float, c_void_p]),
    "seg_relu_dropout_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int64, c_int, c_float, c_uint64, c_void_p, c_void_p]),
    "seg_relu_dropout_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int64, c_int, c_float, c_float, c_void_p]),
    "seg_score_packed_elems": (c_int64, [c_int, c_int]),
    "seg_score_pack": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "seg_score_upsample_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                       c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
    "seg_score_upsample_bwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                       c_int, c_void_p]),
    "seg_score_skip_bwd": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float,
                                   c_void_p]),
    "seg_nhwc_to_nchw_f32": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "seg_axpby_bf16": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int64, c_int, c_float, c_void_p]),
    "seg_comm_buffer_bytes": (ctypes.c_size_t, [c_int, c_int]),
    "seg_comm_alloc": (c_int, [ctypes.c_size_t, POINTER(c_void_p)]),
    "seg_comm_free": (c_int, [c_void_p]),
    "seg_comm_ipc_get": (c_int, [c_void_p, c_void_p]),
    "seg_comm_ipc_open": (c_int, [c_void_p, POINTER(c_void_p)]),
    "seg_comm_ipc_close": (c_int, [c_void_p]),
    "seg_syncbn_exchange": (c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    "seg_sgd_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_float, c_int, c_float, c_void_p]),
    "seg_aug_entry_bytes": (c_int, []),
    "seg_augment_batch_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_float), POINTER(c_float), c_void_p, c_void_p, c_void_p]),
    "seg_aug_scale_entry_bytes": (c_int, []),
    "seg_augment_scale_batch_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_float), POINTER(c_float), c_void_p, c_void_p, c_void_p]),
    "seg_aug_full_entry_bytes": (c_int, []),
    "seg_augment_full_batch_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_float), POINTER(c_float), c_void_p, c_void_p, c_void_p]),
    "seg_augment_val_batch_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_float), POINTER(c_float), c_void_p, c_void_p, c_void_p]),
    "seg_augment_full_blur_batch_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_float), POINTER(c_float), c_void_p,
                                               c_void_p, c_void_p]),
    "seg_resize_nchw_f32": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p]),
    "seg_window_add_nchw_f32": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "seg_div_by_count_nchw_f32": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "seg_argmax_nchw_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "seg_sgd_step_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_float, c_void_p]),
}

EXPORTS = tuple(_SIGS.keys())

_lib = None


def load():
    """Load the shared library (once).  Raises if it has not been built — there is no other code path."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with pytorch-segmentation_b200/build.sh (or __graft_entry__.build()); "
                "the engine has no CPU / eager fallback")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def last_error():
    return load().seg_last_error().decode("utf-8", "replace")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


TRACE = None  # set to a list to record (entry point, meta, start event, end event) for every C-ABI call


def call(name, *args, meta=None):
    """Call ``name`` with the current torch CUDA stream appended; raise RuntimeError on a non-zero status."""
    lib = load()
    if TRACE is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = getattr(lib, name)(*args, stream())
        e1.record()
        TRACE.append((name, meta, e0, e1))
    else:
        rc = getattr(lib, name)(*args, stream())
    if rc != 0:
        raise RuntimeError(f"{name} failed: {last_error()}")


def require_device():
    lib = load()
    if not torch.cuda.is_available():
        raise RuntimeError("seg_b200 needs a CUDA device (sm_90); no CPU fallback exists")
    if lib.seg_device_ok() != 0:
        raise RuntimeError(last_error())


def launch_count():
    return int(load().seg_launch_count())


def reset_launch_count():
    load().seg_launch_count_reset()
