"""Tensor-level front-ends of the C ABI (one function per entry point of include/lwb_b200.h).

Each function checks devices/dtypes/contiguity, allocates outputs with torch (device memory is
torch's job), and calls the library on torch's current stream.  No arithmetic happens here.
"""
import ctypes
import os

import numpy as np
import torch

from . import _lib
from ._lib import ConvDesc, LwbError, check, lib, ptr, stream, _chk_cuda

# utils/nmr.py:177: eye = [0, 0, -(1/tan(30 deg) + 1)], cast to float32 by look_at.py:33
EYE_Z = float(np.float32(-(1. / np.tan(np.radians(30)) + 1)))
NEAR, FAR = 0.1, 100.0              # rasterize.py:10-11 defaults (what render_fim_wim really uses)



def default_align_corners():
    """grid_sample convention of the LWB / source-image warp.  The reference calls F.grid_sample without the flag
    (networks/generator.py:313, models/imitator.py:259) under its pinned torch==1.2.0 (requirements.txt:6), where
    that means align_corners=True; the released checkpoints were trained that way, so True is the default.
    LWB_ALIGN_CORNERS=0 selects what torch >= 1.3 does for the same call."""
    return os.environ.get("LWB_ALIGN_CORNERS", "1") == "1"


_ws_cache = {}

# ---- instrumentation: launch counter (bench.py "gpu_launches") and optional CUDA-event profiling ----
_launches = 0
_profile = None            # None, or {class: [(start_event, end_event, work), ...]}


def reset_launch_count():
    global _launches
    _launches = 0


def launch_count():
    return _launches


def _count(n):
    global _launches
    _launches += n


class _Prof(object):
    """with _Prof('conv', flops): ... -> CUDA events on the launching stream when profiling is on."""

    def __init__(self, cls, work=0.0, label=None):
        self.cls, self.work, self.label = cls, work, label

    def __enter__(self):
        if _profile is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *a):
        if _profile is not None:
            self.e1.record()
            _profile.setdefault(self.cls, []).append((self.e0, self.e1, self.work))
            if self.label:
                _profile.setdefault(self.cls + "/" + self.label, []).append((self.e0, self.e1, self.work))
        return False


def profile_begin():
    global _profile
    _profile = {}


def profile_end():
    """-> {class: {"ms": total, "work": total, "n": launches}}"""
    global _profile
    torch.cuda.synchronize()
    out = {}
    for cls, items in (_profile or {}).items():
        out[cls] = {"ms": sum(a.elapsed_time(b) for a, b, _ in items), "work": sum(w for _, _, w in items), "n": len(items)}
    _profile = None
    return out


def _workspace(nbytes, device):
    key = (device.index, "raster")
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


def raster_forward_face_index_map(faces, face_index_map, weight_map, depth_map, image_size,
                                  near=NEAR, far=FAR, faces_inv=None, flip_rows=False):
    """rasterize_cuda.forward_face_index_map (rasterize_cuda.cpp:70-95): in-place on pre-filled maps."""
    _chk_cuda(faces, face_index_map, weight_map, depth_map, faces_inv)
    if faces.dtype != torch.float32 or face_index_map.dtype != torch.int32 or weight_map.dtype != torch.float32:
        raise LwbError("faces/weight_map must be float32 and face_index_map int32")
    B, F = faces.shape[:2]
    ws = _workspace(lib().lwb_raster_workspace_bytes(B, image_size, F), faces.device)
    check(lib().lwb_raster_forward_face_index_map(
        ptr(faces), B, F, image_size, near, far, ptr(face_index_map), ptr(weight_map), ptr(depth_map),
        ptr(faces_inv), 1 if flip_rows else 0, ptr(ws), stream()), "lwb_raster_forward_face_index_map")
    return face_index_map, weight_map, depth_map


def correspond(cam, verts, face_idx, image_size, map_fn, src_p2verts, src_img=None, align_corners=None,
               want_f2verts=False, near=NEAR, far=FAR, out=None):
    """Fused render_fim_wim + encode_fim + cal_bc_transform + image warp + concat (lwb_correspond).

    -> dict(fim i32[B,H,W], wim f32[B,H,W,3], T f32[B,H,W,2], tsf_inputs f32[B,3+C,H,W],
            tsf_img / cond = channel views of tsf_inputs, f2verts f32[B,F,3,3] | None)
    """
    _chk_cuda(cam, verts, face_idx, map_fn, src_p2verts, src_img)
    if align_corners is None:
        align_corners = default_align_corners()
    B, V = verts.shape[:2]
    F = face_idx.shape[0]
    C = map_fn.shape[1]
    if face_idx.dtype != torch.int32:
        raise LwbError("face_idx must be int32")
    if map_fn.shape[0] != F + 1:
        raise LwbError("map_fn must have F+1 rows (background last)")
    sb = src_p2verts.shape[0]
    dev = verts.device
    s = image_size
    if out is None:
        out = dict(fim=torch.empty((B, s, s), dtype=torch.int32, device=dev),
                   wim=torch.empty((B, s, s, 3), dtype=torch.float32, device=dev),
                   T=torch.empty((B, s, s, 2), dtype=torch.float32, device=dev),
                   tsf_inputs=torch.empty((B, 3 + C, s, s), dtype=torch.float32, device=dev),
                   f2verts=torch.empty((B, F, 3, 3), dtype=torch.float32, device=dev) if want_f2verts else None)
    ws = _workspace(lib().lwb_raster_workspace_bytes(B, s, F), dev)
    _count(3)
    # algorithmic bytes (SURVEY.md 8d): per frame verts + fim/wim/T/tsf_inputs; per batch the shared tables
    nbytes = B * (V * 12 + s * s * (4 + 12 + 8 + 4 * (3 + C))) + F * 12 + sb * F * 24 + (F + 1) * C * 4 + sb * 3 * s * s * 4
    with _Prof("correspond", nbytes):
      check(lib().lwb_correspond(
        ptr(cam), ptr(verts), ptr(face_idx), B, V, F, s, near, far, EYE_Z,
        ptr(map_fn), C, ptr(src_p2verts), ptr(src_img), sb, 1 if align_corners else 0,
        ptr(out["fim"]), ptr(out["wim"]), ptr(out["T"]), ptr(out["tsf_inputs"]), ptr(out.get("f2verts")),
        ptr(ws), stream()), "lwb_correspond")
    out["tsf_img"] = out["tsf_inputs"][:, :3]
    out["cond"] = out["tsf_inputs"][:, 3:]
    return out


def warp_nchw(x, T, align_corners=None, out=None, accumulate=False):
    """transform / stn (networks/generator.py:303-320): x [Bs,C,h,w], T [B,TH,TW,2] -> [B,C,h,w]."""
    _chk_cuda(x, T, out)
    if align_corners is None:
        align_corners = default_align_corners()
    if x.dtype != torch.float32 or T.dtype != torch.float32:
        raise LwbError("warp expects float32")
    sb, C, h, w = x.shape
    B, th, tw = T.shape[:3]
    if out is None:
        out = torch.empty((B, C, h, w), dtype=torch.float32, device=x.device)
    check(lib().lwb_warp_nchw(ptr(x), sb, C, h, w, ptr(T), B, th, tw, 1 if align_corners else 0,
                              ptr(out), 1 if accumulate else 0, stream()), "lwb_warp_nchw")
    return out


class PackedWeight(tuple):
    """(hi, lo) operand tensors of one conv layer; ``w_exp`` = the power of two they were packed with (every split)."""

    def __new__(cls, hi, lo, w_exp):
        self = super(PackedWeight, cls).__new__(cls, (hi, lo))
        self.w_exp = w_exp
        return self


def weight_exponent(absmax):
    """Per-layer scale of the weight packing in every operand mode: E with absmax * 2^E in [2^14, 2^15) (15 for an
    all-zero layer).  It keeps the fp16 hi / lo weights of small-weight layers out of the fp16 subnormals."""
    import math
    absmax = float(absmax)
    if not (absmax > 0.0) or math.isinf(absmax) or math.isnan(absmax):
        return 15
    return max(-40, min(60, 15 - math.frexp(absmax)[1]))


def pack_conv_weight(w, transposed=False, cout_pad=None, cin_pad=None, split=True, absmax=None):
    """OIHW / IOHW fp32 -> ([tap][cout_pad][cin_pad] fp16 hi, lo) of w x 2^w_exp.  split: 0/False single, 1/True fp16
    hi+lo, 2 fp16 hi + fp8 pair blocks (lwb_pack_conv_weight_f8).  ``absmax`` = max|w| when the caller already knows it
    (one host sync per network instead of one per layer); computed here otherwise."""
    _chk_cuda(w)
    if int(split) == 2:
        return _pack_conv_weight_f8(w, transposed, cout_pad, cin_pad, absmax)
    w = w.float().contiguous()
    if transposed:
        cin, cout, kh, kw = w.shape
    else:
        cout, cin, kh, kw = w.shape
    cout_pad = cout_pad or cout
    cin_pad = cin_pad or cin
    w_exp = weight_exponent(w.abs().max() if absmax is None else absmax)
    hi = torch.empty((kh * kw, cout_pad, cin_pad), dtype=torch.float16, device=w.device)
    lo = torch.empty_like(hi) if split else None
    check(lib().lwb_pack_conv_weight(ptr(w), cout, cin, kh, kw, 1 if transposed else 0, cout_pad, cin_pad, w_exp,
                                     ptr(hi), ptr(lo), stream()), "lwb_pack_conv_weight")
    return PackedWeight(hi, lo, w_exp)


def _pack_conv_weight_f8(w, transposed, cout_pad, cin_pad, absmax=None):
    w = w.float().contiguous()
    if transposed:
        cin, cout, kh, kw = w.shape
    else:
        cout, cin, kh, kw = w.shape
    cout_pad = cout_pad or cout
    cin_pad = cin_pad or cin
    w_exp = weight_exponent(w.abs().max() if absmax is None else absmax)
    hi = torch.empty((kh * kw, cout_pad, cin_pad), dtype=torch.float16, device=w.device)
    lo = torch.empty_like(hi)                                   # same bytes, fp8 pair blocks inside
    check(lib().lwb_pack_conv_weight_f8(ptr(w), cout, cin, kh, kw, 1 if transposed else 0, cout_pad, cin_pad, w_exp,
                                        ptr(hi), ptr(lo), stream()), "lwb_pack_conv_weight_f8")
    return PackedWeight(hi, lo, w_exp)


def pack_conv_weight_rowk(w, cout_pad=None, cpx=8, kxs=8, split=True, absmax=None):
    """7x7 stem weights -> [ky][cout_pad][kxs*cpx] fp16 hi, lo of w x 2^w_exp (K index = kx*cpx + c)."""
    _chk_cuda(w)
    w = w.float().contiguous()
    cout, cin, kh, kw = w.shape
    cout_pad = cout_pad or cout
    w_exp = weight_exponent(w.abs().max() if absmax is None else absmax)
    hi = torch.empty((kh, cout_pad, kxs * cpx), dtype=torch.float16, device=w.device)
    lo = torch.empty_like(hi) if split else None
    check(lib().lwb_pack_conv_weight_rowk(ptr(w), cout, cin, kh, kw, cout_pad, cpx, kxs, w_exp, ptr(hi), ptr(lo),
                                          stream()), "lwb_pack_conv_weight_rowk")
    return PackedWeight(hi, lo, w_exp)


def nchw_to_nhwc_split(x, c_pad=None, pad_hw=(0, 0, 0, 0), hi=None, lo=None, split=True):
    """NCHW fp32 -> NHWC fp16 hi/lo [n, h+top+bottom, w+left+right, c_pad]; pad_hw = (top, bottom, left, right)."""
    _chk_cuda(x, hi, lo)
    n, c, h, w = x.shape
    c_pad = c_pad or c
    top, bottom, left, right = pad_hw
    hp, wp = h + top + bottom, w + left + right
    if hi is None:
        hi = torch.empty((n, hp, wp, c_pad), dtype=torch.float16, device=x.device)
        lo = torch.empty_like(hi) if split else None
    _count(1)
    with _Prof("input", n * c * h * w * 4 + n * hp * wp * c_pad * (4 if lo is not None else 2)):
        check(lib().lwb_nchw_to_nhwc_split(ptr(x), n, c, h, w, c_pad, hp, wp, top, left, ptr(hi), ptr(lo), stream()),
              "lwb_nchw_to_nhwc_split")
    return hi, lo


def nhwc_to_nchw(x, c=None, out=None):
    _chk_cuda(x, out)
    n, h, w, cs = x.shape
    c = c or cs
    if out is None:
        out = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    check(lib().lwb_nhwc_to_nchw(ptr(x), n, c, h, w, cs, ptr(out), stream()), "lwb_nhwc_to_nchw")
    return out


class ConvPlan(object):
    """One conv layer bound to fixed buffers (lwb_conv_plan): build once, run every step."""

    def __init__(self, desc, x0, x1, w, out_raw, stats):
        """x0 / x1 / w: (hi, lo) tensor pairs (x1 may be None), w a PackedWeight; out_raw fp32 NHWC; stats f64
        [n,cout,2] or None."""
        self._keep = (x0, x1, w, out_raw, stats)
        self.desc = desc
        desc.w_exp = int(w.w_exp)
        handle = ctypes.c_void_p()
        x1 = x1 or (None, None)
        check(lib().lwb_conv_plan_create(ctypes.byref(desc), ptr(x0[0]), ptr(x0[1]), ptr(x1[0]), ptr(x1[1]),
                                         ptr(w[0]), ptr(w[1]), ptr(out_raw), ptr(stats), ctypes.byref(handle)),
              "lwb_conv_plan_create")
        self._h = handle
        self.num_launches = lib().lwb_conv_plan_num_launches(handle)
        d = desc
        self.label = "%s%dx%ds%d %d->%d @%d" % ("T" if d.transposed else ("R" if d.rowk else "C"), d.kh, d.kw, d.stride,
                                                d.cin0 + d.cin1, d.cout, d.h_out)
        if d.transposed:       # algorithmic 2*MAC: every input pixel meets every (tap, cin, cout)
            self.flops = 2.0 * d.n * d.h_in * d.w_in * d.cin0 * d.cout * d.kh * d.kw
        elif d.rowk:
            self.flops = 2.0 * d.n * d.h_out * d.w_out * d.cout * w[0].shape[0] * 7 * getattr(self, "_real_cin", 6)
        else:
            self.flops = 2.0 * d.n * d.h_out * d.w_out * d.cout * (d.cin0 + d.cin1) * d.kh * d.kw

    prof_class = "conv"                  # instrumentation class (bench.py breakdown); the folded heads report as "heads"

    def run(self):
        _count(self.num_launches)
        with _Prof(self.prof_class, self.flops, self.label):
            check(lib().lwb_conv_plan_run(self._h, stream()), "lwb_conv_plan_run")

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().lwb_conv_plan_destroy(self._h)
                self._h = None
        except Exception:
            pass


def make_conv_desc(n, h_in, w_in, cin0, cout, kh, kw, stride=1, pad=0, dil=1, cin1=0, transposed=False,
                   split=True, rowk=False, row_pitch=0, n_tile=0, halo=False, pad_w=None):
    if transposed:
        h_out, w_out = 2 * h_in, 2 * w_in
    elif rowk:
        h_out, w_out = h_in, w_in
    else:
        h_out = (h_in + 2 * pad - dil * (kh - 1) - 1) // stride + 1
        w_out = (w_in + 2 * (pad if pad_w is None else pad_w) - dil * (kw - 1) - 1) // stride + 1
    return ConvDesc(w_exp=15, pad_w=-1 if pad_w is None else pad_w, n=n, h_in=h_in, w_in=w_in, h_out=h_out, w_out=w_out, cin0=cin0, cin1=cin1, cout=cout,
                    kh=kh, kw=kw, stride=stride, pad=pad, dil=dil, transposed=1 if transposed else 0,
                    split=int(split), rowk=1 if rowk else 0, row_pitch=row_pitch, n_tile=n_tile,
                    halo=1 if halo else 0)


def instance_stats_nhwc(x, stats=None):
    _chk_cuda(x, stats)
    n, h, w, c = x.shape
    if stats is None:
        stats = torch.zeros((n, c, 2), dtype=torch.float64, device=x.device)
    check(lib().lwb_instance_stats_nhwc(ptr(x), n, h, w, c, ptr(stats), stream()), "lwb_instance_stats_nhwc")
    return stats


def norm_act_nhwc(raw, stats, gamma, beta, relu, ws, eps=1e-5, residual=None, warp_src=None, T=None,
                  align_corners=False, y_f32=None, y_hi=None, y_lo=None, lo_format=0,
                  post_scale=None, post_shift=None, post_relu=False, res_step=1, range_flag=None):
    """InstanceNorm + ReLU + residual + LWB warp-add on an NHWC fp32 tensor (lwb_norm_act_nhwc).
    lo_format 1: y_lo receives the fp8 pair blocks that split=2 conv plans consume.  stats=None with gamma/beta: plain
    per-channel affine (folded BatchNorm / bias); post_*: second affine (+ReLU) applied to the operands only;
    res_step: subsampled residual; range_flag: int32[1] device tensor collecting the operand-range bits."""
    _chk_cuda(raw, stats, gamma, beta, residual, warp_src, T, ws, y_f32, y_hi, y_lo, post_scale, post_shift, range_flag)
    n, h, w, c = raw.shape
    sb, th, tw = 0, 0, 0
    if warp_src is not None:
        sb = warp_src.shape[0]
        th, tw = T.shape[1:3]
    _count(2 if (stats is not None or gamma is not None or beta is not None) else 1)
    per = 4 + (4 if residual is not None else 0) + (4 if y_f32 is not None else 0) \
        + (2 if y_hi is not None else 0) + (2 if y_lo is not None else 0)
    nbytes = n * h * w * c * per + (warp_src.numel() * 4 + n * h * w * 8 if warp_src is not None else 0)
    with _Prof("norm", nbytes, "%dx%d c%d%s%s" % (h, w, c, " +res" if residual is not None else "", " +warp" if warp_src is not None else "")):
        check(lib().lwb_norm_act_nhwc(ptr(raw), ptr(stats), ptr(gamma), ptr(beta), eps, 1 if relu else 0, n, h, w, c,
                                      ptr(residual), ptr(warp_src), sb, ptr(T), th, tw, 1 if align_corners else 0,
                                      ptr(ws), ptr(y_f32), ptr(y_hi), ptr(y_lo), int(lo_format),
                                      ptr(post_scale), ptr(post_shift), 1 if post_relu else 0, int(res_step),
                                      ptr(range_flag), stream()), "lwb_norm_act_nhwc")


def pack_head_weights(w_img, w_att):
    _chk_cuda(w_img, w_att)
    w4 = torch.empty((49, 64, 4), dtype=torch.float32, device=w_img.device)
    check(lib().lwb_pack_head_weights(ptr(w_img.float().contiguous()), ptr(w_att.float().contiguous()), ptr(w4), stream()),
          "lwb_pack_head_weights")
    return w4


def conv7x7_heads_nhwc(x, w4, out=None):
    _chk_cuda(x, w4, out)
    n, h, w, c = x.shape
    if c != 64:
        raise LwbError("heads expect 64 input channels")
    if out is None:
        out = torch.empty((n, h, w, 4), dtype=torch.float32, device=x.device)
    _count(1)
    with _Prof("heads", 2.0 * n * h * w * 49 * 64 * 4):
        check(lib().lwb_conv7x7_heads_nhwc(ptr(x), ptr(w4), n, h, w, ptr(out), stream()), "lwb_conv7x7_heads_nhwc")
    return out


def heads_composite(raw, bg=None, want_color=True, want_mask=True, color=None, mask=None, pred=None,
                    want_pred=True, pred_hwc=None, pred_u8=None, folded_kw=0, range_flag=None):
    """-> color, mask, pred (NCHW).  ``pred_hwc`` f32 [n,h,w,3] / ``pred_u8`` uint8 BGR [n,h,w,3]: caller-allocated
    output-path buffers filled by the same launch."""
    _chk_cuda(raw, bg, color, mask, pred, pred_hwc, pred_u8)
    n, h, w, cs = raw.shape
    dev = raw.device
    if color is None and want_color:
        color = torch.empty((n, 3, h, w), dtype=torch.float32, device=dev)
    if mask is None and want_mask:
        mask = torch.empty((n, 1, h, w), dtype=torch.float32, device=dev)
    if pred is None and bg is not None and want_pred:
        pred = torch.empty((n, 3, h, w), dtype=torch.float32, device=dev)
    for t, dt in ((pred_hwc, torch.float32), (pred_u8, torch.uint8)):
        if t is not None and (t.dtype != dt or tuple(t.shape) != (n, h, w, 3)):
            raise LwbError("output-path buffers must be [n,h,w,3] float32 / uint8")
    _count(1)
    with _Prof("heads", 0.0):
        check(lib().lwb_heads_composite(ptr(raw), n, h, w, cs, int(folded_kw), ptr(bg), bg.shape[0] if bg is not None else 0,
                                        ptr(color), ptr(mask), ptr(pred), ptr(pred_hwc), ptr(pred_u8), ptr(range_flag), stream()),
              "lwb_heads_composite")
    return color, mask, pred


def frames_out(frames, want_hwc=True, want_u8=False):
    """[n,3,h,w] fp32 -> (hwc f32 [n,h,w,3] | None, u8 BGR [n,h,w,3] | None): models/imitator.py:178-180 +
    utils/cv_utils.py:23-36."""
    _chk_cuda(frames)
    n, c, h, w = frames.shape
    if c != 3 or frames.dtype != torch.float32:
        raise LwbError("frames must be float32 [n,3,h,w]")
    hwc = torch.empty((n, h, w, 3), dtype=torch.float32, device=frames.device) if want_hwc else None
    u8 = torch.empty((n, h, w, 3), dtype=torch.uint8, device=frames.device) if want_u8 else None
    _count(1)
    check(lib().lwb_frames_out(ptr(frames), n, h, w, ptr(hwc), ptr(u8), stream()), "lwb_frames_out")
    return hwc, u8


def conv2d_direct_nchw(x, w, bias=None, stride=1, pad=0, dil=1):
    _chk_cuda(x, w, bias)
    n, cin, h, wd = x.shape
    cout, _, kh, kw = w.shape
    ho = (h + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    wo = (wd + 2 * pad - dil * (kw - 1) - 1) // stride + 1
    out = torch.empty((n, cout, ho, wo), dtype=torch.float32, device=x.device)
    check(lib().lwb_conv2d_direct_nchw(ptr(x), ptr(w), ptr(bias), n, cin, h, wd, cout, kh, kw, stride, pad, dil,
                                       ptr(out), stream()), "lwb_conv2d_direct_nchw")
    return out


def gated_act_nhwc(raw, c, bias, act, scale, shift, upsample=1, clamp=False, y_f32=None, y_hi=None, y_lo=None,
                   lo_format=0, range_flag=None):
    """Gated-conv epilogue on the conv engine's raw NHWC output [n,h,w,c_stride >= 2c] (lwb_gated_act_nhwc):
    y = BN(act(a + bias_a) * sigmoid(b + bias_b)) -> optional fp32 [n,h*u,w*u,*] and the next layer's operands
    [n,h*u,w*u,c_pad] (zero-padded channels), on the 2x nearest-neighbour grid when upsample = 2."""
    _chk_cuda(raw, bias, scale, shift, y_f32, y_hi, y_lo, range_flag)
    n, h, w, cs = raw.shape
    u = int(upsample)
    for t in (y_f32, y_hi):
        if t is not None and tuple(t.shape[:3]) != (n, h * u, w * u):
            raise LwbError("gated_act: output grid must be [n, %d, %d, *]" % (h * u, w * u))
    _count(1)
    check(lib().lwb_gated_act_nhwc(ptr(raw), n, h, w, int(c), cs, ptr(bias), int(act), ptr(scale), ptr(shift), u, 1 if clamp else 0,
                                   ptr(y_f32), y_f32.shape[3] if y_f32 is not None else 0, ptr(y_hi), ptr(y_lo),
                                   y_hi.shape[3] if y_hi is not None else 0, int(lo_format), ptr(range_flag), stream()),
          "lwb_gated_act_nhwc")


def self_attention_nhwc(qkv, bias, x, gamma, dq=16, out=None):
    """SelfAttention (networks/inpaintor.py:86-107): qkv [n,h,w,ld] = [q | k | v | pad] raw 1x1-conv output, bias
    [2*dq+dv], x [n,h,w,dv] fp32 -> gamma * softmax(q k^T) v + x."""
    _chk_cuda(qkv, bias, x, gamma, out)
    n, h, w, ld = qkv.shape
    dv = x.shape[3]
    if out is None:
        out = torch.empty_like(x)
    _count(1)
    check(lib().lwb_self_attention_nhwc(ptr(qkv), ld, ptr(bias), n, h * w, int(dq), dv, ptr(x), ptr(gamma), ptr(out), stream()),
          "lwb_self_attention_nhwc")
    return out


def maxpool_nchw_to_nhwc(x, k, stride, out=None):
    """F.max_pool2d(x, k, stride, ceil_mode=True) (networks/hmr.py:150): NCHW fp32 -> NHWC fp32."""
    _chk_cuda(x, out)
    n, c, h, w = x.shape
    ho, wo = -(-(h - k) // stride) + 1, -(-(w - k) // stride) + 1
    if out is None:
        out = torch.empty((n, ho, wo, c), dtype=torch.float32, device=x.device)
    _count(1)
    check(lib().lwb_maxpool_nchw_to_nhwc(ptr(x), n, c, h, w, k, stride, ptr(out), stream()), "lwb_maxpool_nchw_to_nhwc")
    return out


def global_avgpool_nhwc(x, scale=None, shift=None, relu=False, out=None, ld_out=None):
    """mean over pixels of relu?(x*scale+shift): x NHWC fp32 [n,h,w,c] -> out [n, ld_out] (first c columns)."""
    _chk_cuda(x, scale, shift)
    n, h, w, c = x.shape
    if out is None:
        out = torch.empty((n, c), dtype=torch.float32, device=x.device)
    ld = ld_out if ld_out is not None else out.stride(0)
    _count(1)
    check(lib().lwb_global_avgpool_nhwc(ptr(x), n, h * w, c, ptr(scale), ptr(shift), 1 if relu else 0, ptr(out), ld, stream()),
          "lwb_global_avgpool_nhwc")
    return out


def linear(x, w, bias=None, relu=False, out=None, accumulate=False):
    """nn.Linear (+ReLU): x [n,k] (row stride x.stride(0)), w [m,k] -> out [n,m] (row stride out.stride(0)), += if accumulate."""
    _chk_cuda(w, bias)
    for t in (x, out):
        if t is not None and (not t.is_cuda or t.stride(-1) != 1):
            raise LwbError("linear expects CUDA tensors with unit inner stride")
    n, k = x.shape
    m = w.shape[0]
    if w.shape[1] != k:
        raise LwbError("linear: weight is [%d,%d], input has %d features" % (m, w.shape[1], k))
    if out is None:
        out = torch.empty((n, m), dtype=torch.float32, device=x.device)
    _count(1)
    check(lib().lwb_linear(ptr(x), x.stride(0), ptr(w), ptr(bias), n, k, m, 1 if relu else 0, 1 if accumulate else 0,
                           ptr(out), out.stride(0), stream()), "lwb_linear")
    return out


def gated_bn_nchw(ab, act, scale=None, shift=None):
    """networks/inpaintor.py:37-47: act(a)*sigmoid(b) followed by folded eval-mode BatchNorm."""
    _chk_cuda(ab, scale, shift)
    n, c2, h, w = ab.shape
    out = torch.empty((n, c2 // 2, h, w), dtype=torch.float32, device=ab.device)
    check(lib().lwb_gated_bn_nchw(ptr(ab), n, c2 // 2, h, w, act, ptr(scale), ptr(shift), ptr(out), stream()),
          "lwb_gated_bn_nchw")
    return out


def smpl_forward(beta, theta, model, rotate_base=False, cam=None, want_joints=True):
    """SMPL.forward (networks/batch_smpl.py:285-375) through lwb_smpl_forward.  ``model``: dict of device
    tensors (see impersonator_b200.smpl.SMPL._device_model).  -> verts [B,V,3], joints [B,NJ,3] | None,
    Rs [B,24,3,3], J_transformed [B,24,3], j2d [B,NJ,2] | None."""
    _chk_cuda(beta, theta, cam)
    if beta.dtype != torch.float32 or theta.dtype != torch.float32:
        raise LwbError("beta/theta must be float32")
    B = beta.shape[0]
    if theta.shape != (B, 72):
        raise LwbError("theta must be [B,72]")
    dev = beta.device
    V = model["v_template"].shape[0]
    nb = model["shapedirs"].shape[0]
    if beta.shape[1] != nb:
        raise LwbError("beta must be [B,%d]" % nb)
    nj = model["joint_regressor_t"].shape[0]
    verts = torch.empty(B, V, 3, dtype=torch.float32, device=dev)
    Rs = torch.empty(B, 24, 3, 3, dtype=torch.float32, device=dev)
    Jt = torch.empty(B, 24, 3, dtype=torch.float32, device=dev)
    joints = torch.empty(B, nj, 3, dtype=torch.float32, device=dev) if want_joints else None
    j2d = torch.empty(B, nj, 2, dtype=torch.float32, device=dev) if (want_joints and cam is not None) else None
    key = (dev.index, "smpl")
    n = lib().lwb_smpl_workspace_bytes(B)
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < n:
        ws = _ws_cache[key] = torch.empty(n, dtype=torch.uint8, device=dev)
    check(lib().lwb_smpl_forward(
        ptr(beta), ptr(theta), B, nb, V, ptr(model["v_template"]), ptr(model["shapedirs"]), ptr(model["posedirs"]),
        ptr(model["j_template"]), ptr(model["j_shapedirs"]), ptr(model["parents"]), ptr(model["weights"]),
        ptr(model["joint_regressor_t"]), nj, 1 if rotate_base else 0,
        ptr(verts), ptr(joints), ptr(Rs), ptr(Jt), ptr(cam if j2d is not None else None), ptr(j2d), ptr(ws), stream()),
        "lwb_smpl_forward")
    _count(3 if want_joints else 2)
    return verts, joints, Rs, Jt, j2d
