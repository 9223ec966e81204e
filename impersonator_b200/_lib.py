"""ctypes binding of the C-ABI library ``liblwb_b200.so`` (include/lwb_b200.h).

The library is the product: there is NO Python/torch fallback.  If the shared object is missing
or a call fails, an exception is raised (``LwbError``) -- loudly, as the parity claims require.
Torch is used only for device memory, streams and dtype bookkeeping; every signature below is
plain pointers + ints.
"""
import ctypes
import os
import subprocess

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblwb_b200.so")
CSRC = os.path.join(_HERE, "csrc")


class LwbError(RuntimeError):
    pass


class ConvDesc(ctypes.Structure):
    """struct lwb_conv_desc (include/lwb_b200.h)."""
    _fields_ = [(n, ctypes.c_int) for n in (
        "n", "h_in", "w_in", "h_out", "w_out", "cin0", "cin1", "cout",
        "kh", "kw", "stride", "pad", "dil", "transposed", "split", "rowk", "row_pitch", "n_tile", "halo", "w_exp", "pad_w")]


_vp, _i, _f, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t

# name -> (restype, argtypes); must list EVERY symbol include/lwb_b200.h declares (tests check it).
SIGNATURES = {
    "lwb_version": (_i, []),
    "lwb_last_error": (ctypes.c_char_p, []),
    "lwb_device_info": (_i, [_vp, _vp, _vp]),
    "lwb_raster_workspace_bytes": (_sz, [_i, _i, _i]),
    "lwb_raster_forward_face_index_map": (_i, [_vp, _i, _i, _i, _f, _f, _vp, _vp, _vp, _vp, _i, _vp, _vp]),
    "lwb_correspond": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _f, _f, _f, _vp, _i, _vp, _vp, _i, _i,
                            _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "lwb_warp_nchw": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _vp, _i, _vp]),
    "lwb_pack_conv_weight": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "lwb_pack_conv_weight_f8": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "lwb_pack_conv_weight_rowk": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "lwb_nchw_to_nhwc_split": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "lwb_nhwc_to_nchw": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "lwb_conv_plan_create": (_i, [ctypes.POINTER(ConvDesc), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                  ctypes.POINTER(_vp)]),
    "lwb_conv_plan_run": (_i, [_vp, _vp]),
    "lwb_conv_plan_num_launches": (_i, [_vp]),
    "lwb_conv_plan_destroy": (None, [_vp]),
    "lwb_conv2d_nhwc": (_i, [ctypes.POINTER(ConvDesc), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "lwb_instance_stats_nhwc": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "lwb_norm_act_nhwc": (_i, [_vp, _vp, _vp, _vp, _f, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _i, _i, _i,
                               _vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _vp, _vp]),
    "lwb_pack_head_weights": (_i, [_vp, _vp, _vp, _vp]),
    "lwb_conv7x7_heads_nhwc": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "lwb_heads_composite": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "lwb_frames_out": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    "lwb_gated_bn_nchw": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "lwb_smpl_workspace_bytes": (_sz, [_i]),
    "lwb_smpl_forward": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i,
                              _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "lwb_gated_act_nhwc": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _vp]),
    "lwb_self_attention_nhwc": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "lwb_maxpool_nchw_to_nhwc": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "lwb_global_avgpool_nhwc": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _i, _vp]),
    "lwb_linear": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _vp, _i, _vp]),
    "lwb_conv2d_direct_nchw": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "lwb_conv2d_direct_relu_nhwc": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "lwb_maxpool_nhwc": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "lwb_ssim_psnr_workspace_bytes": (_sz, [_i, _i, _i]),
    "lwb_ssim_psnr": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "lwb_lpips_input": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "lwb_lpips_layer": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp]),
    "lwb_inception_input": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "lwb_bn_act_segment": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _vp]),
    "lwb_maxpool_nhwc_slice": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _vp]),
    "lwb_det_transform": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "lwb_det_stem_pool": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "lwb_det_bias_act": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "lwb_det_d2s_bias_relu": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "lwb_det_rpn": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _f, _f, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp]),
    "lwb_det_nms_workspace_bytes": (_sz, [_i, _i]),
    "lwb_det_nms": (_i, [_vp, _vp, _vp, _vp, _i, _i, _f, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "lwb_det_roi_align": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "lwb_det_box_candidates": (_i, [_vp, _i, _i, _vp, _vp, _i, _f, _f, _f, _f, _f, _vp, _vp, _vp, _vp, _vp]),
    "lwb_det_mask_probs": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "lwb_det_paste_masks": (_i, [_vp, _i, _vp, _vp, _i, _f, _f, _i, _i, _vp, _vp, _vp]),
    "lwb_det_person_mask": (_i, [_vp, _vp, _vp, _i, _vp, _i, _i, _f, _i, _vp, _vp, _vp, _vp]),
}

_lib = None


def build(verbose=False):
    """Compile every CUDA source for sm_90a into impersonator_b200/liblwb_b200.so (nvcc, in-tree)."""
    out = subprocess.run(["make", "-C", CSRC, "-j8"], capture_output=True, text=True)
    if verbose or out.returncode != 0:
        print(out.stdout[-4000:], out.stderr[-4000:])
    if out.returncode != 0:
        raise LwbError("building liblwb_b200.so failed")
    return LIB_PATH


def lib():
    """Load the C-ABI library (no GPU needed to load).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LwbError("%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU/torch fallback)" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)          # AttributeError if a declared symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc, what=""):
    if rc != 0:
        raise LwbError("%s failed (%d): %s" % (what, rc, lib().lwb_last_error().decode()))


def require_gpu():
    """Fail loudly unless a sm_90 device is current (the kernels are sm_90a-only)."""
    if not torch.cuda.is_available():
        raise LwbError("no CUDA device: the lwb_b200 path has no CPU fallback")
    sm, ma, mi = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    check(lib().lwb_device_info(ctypes.byref(sm), ctypes.byref(ma), ctypes.byref(mi)), "lwb_device_info")
    if (ma.value, mi.value) != (9, 0):
        raise LwbError("device is sm_%d%d; this library is built for sm_90a only" % (ma.value, mi.value))
    return sm.value


def ptr(t):
    return 0 if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def _chk_cuda(*ts):
    cur = None
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise LwbError("expected a CUDA tensor (no CPU path)")
        if not t.is_contiguous():
            raise LwbError("expected a contiguous tensor")
        if cur is None:
            cur = torch.cuda.current_device()
        if t.device.index != cur:
            # the launch goes to the CURRENT device's stream: refuse instead of launching on the wrong GPU
            raise LwbError("tensor lives on cuda:%d but the current device is cuda:%d: wrap the call in "
                           "torch.cuda.device(%d) / torch.cuda.set_device" % (t.device.index, cur, t.device.index))
