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


def _workspace(nbytes, device, kind):
    """The device's cached ``kind`` workspace, grown to ``nbytes``.  Pinned to the CUDA graphs being captured: a larger
    call replaces the cached buffer, and a graph must not replay into one the allocator has handed to another tensor."""
    key = (device.index, kind)
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return _lib.pin(buf)


def _chk_tensor(name, t, dtype, shape):
    """Raise unless ``t`` has ``dtype`` and ``shape`` (None in ``shape``: any size)."""
    if t.dtype != dtype or t.dim() != len(shape) or any(s is not None and t.shape[i] != s for i, s in enumerate(shape)):
        raise LwbError("%s must be %s %s, got %s %s" % (name, str(dtype).replace("torch.", ""),
                                                        list("*" if s is None else s for s in shape),
                                                        str(t.dtype).replace("torch.", ""), list(t.shape)))


def raster_forward_face_index_map(faces, face_index_map, weight_map, depth_map, image_size,
                                  near=NEAR, far=FAR, faces_inv=None, flip_rows=False):
    """rasterize_cuda.forward_face_index_map (rasterize_cuda.cpp:70-95): in-place on pre-filled maps.  Only covered pixels
    are written; depth_map and faces_inv may be None."""
    _chk_cuda(faces, face_index_map, weight_map, depth_map, faces_inv)
    _chk_tensor("faces", faces, torch.float32, (None, None, 3, 3))
    B, F = faces.shape[:2]
    s = image_size
    _chk_tensor("face_index_map", face_index_map, torch.int32, (B, s, s))
    _chk_tensor("weight_map", weight_map, torch.float32, (B, s, s, 3))
    if depth_map is not None:
        _chk_tensor("depth_map", depth_map, torch.float32, (B, s, s))
    if faces_inv is not None:
        _chk_tensor("faces_inv", faces_inv, torch.float32, (B, F, 3, 3))
    ws = _workspace(lib().lwb_raster_workspace_bytes(B, image_size, F), faces.device, "raster")
    check(lib().lwb_raster_forward_face_index_map(
        ptr(faces), B, F, image_size, near, far, ptr(face_index_map), ptr(weight_map), ptr(depth_map),
        ptr(faces_inv), 1 if flip_rows else 0, ptr(ws), stream()), "lwb_raster_forward_face_index_map")
    return face_index_map, weight_map, depth_map


def correspond(cam, verts, face_idx, image_size, map_fn, src_p2verts, src_img=None, align_corners=None,
               want_f2verts=False, near=NEAR, far=FAR, out=None):
    """Fused render_fim_wim + encode_fim + cal_bc_transform + image warp + concat (lwb_correspond).

    cam f32[B,3], verts f32[B,V,3], face_idx i32[F,3], map_fn f32[F+1,C] (background row last), src_p2verts f32[sb,F,3,2]
    and src_img None | f32[sb,3,H,W] with sb = 1 (one source for every frame) or B.  ``out``: caller buffers of the shapes
    below (f2verts may be None).
    -> dict(fim i32[B,H,W], wim f32[B,H,W,3], T f32[B,H,W,2], tsf_inputs f32[B,3+C,H,W],
            tsf_img / cond = channel views of tsf_inputs, f2verts f32[B,F,3,3] | None)
    """
    _chk_cuda(cam, verts, face_idx, map_fn, src_p2verts, src_img)
    if align_corners is None:
        align_corners = default_align_corners()
    _chk_tensor("verts", verts, torch.float32, (None, None, 3))
    B, V = verts.shape[:2]
    s = image_size
    _chk_tensor("cam", cam, torch.float32, (B, 3))
    _chk_tensor("face_idx", face_idx, torch.int32, (None, 3))
    F = face_idx.shape[0]
    _chk_tensor("map_fn (F+1 rows, background last)", map_fn, torch.float32, (F + 1, None))
    C = map_fn.shape[1]
    _chk_tensor("src_p2verts", src_p2verts, torch.float32, (None, F, 3, 2))
    sb = src_p2verts.shape[0]
    if sb not in (1, B):
        raise LwbError("src_p2verts has %d sources for %d frames: 1 or B" % (sb, B))
    if src_img is not None:
        _chk_tensor("src_img", src_img, torch.float32, (sb, 3, s, s))
    dev = verts.device
    if out is None:
        out = dict(fim=torch.empty((B, s, s), dtype=torch.int32, device=dev),
                   wim=torch.empty((B, s, s, 3), dtype=torch.float32, device=dev),
                   T=torch.empty((B, s, s, 2), dtype=torch.float32, device=dev),
                   tsf_inputs=torch.empty((B, 3 + C, s, s), dtype=torch.float32, device=dev),
                   f2verts=torch.empty((B, F, 3, 3), dtype=torch.float32, device=dev) if want_f2verts else None)
    else:
        _chk_cuda(out["fim"], out["wim"], out["T"], out["tsf_inputs"], out.get("f2verts"))
        _chk_tensor("out['fim']", out["fim"], torch.int32, (B, s, s))
        _chk_tensor("out['wim']", out["wim"], torch.float32, (B, s, s, 3))
        _chk_tensor("out['T']", out["T"], torch.float32, (B, s, s, 2))
        _chk_tensor("out['tsf_inputs']", out["tsf_inputs"], torch.float32, (B, 3 + C, s, s))
        if out.get("f2verts") is not None:
            _chk_tensor("out['f2verts']", out["f2verts"], torch.float32, (B, F, 3, 3))
    ws = _workspace(lib().lwb_raster_workspace_bytes(B, s, F), dev, "raster")
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
    w = w.float().contiguous()
    if transposed:
        cin, cout, kh, kw = w.shape
    else:
        cout, cin, kh, kw = w.shape
    cout_pad = cout_pad or cout
    cin_pad = cin_pad or cin
    w_exp = weight_exponent(w.abs().max() if absmax is None else absmax)
    hi = torch.empty((kh * kw, cout_pad, cin_pad), dtype=torch.float16, device=w.device)
    lo = torch.empty_like(hi) if split else None                # split 2: same bytes, fp8 pair blocks inside
    entry = "lwb_pack_conv_weight_f8" if int(split) == 2 else "lwb_pack_conv_weight"
    check(getattr(lib(), entry)(ptr(w), cout, cin, kh, kw, 1 if transposed else 0, cout_pad, cin_pad, w_exp,
                                ptr(hi), ptr(lo), stream()), entry)
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

    def launch_info(self, i=0):
        """-> dict(n_tile, mode, k_stages, taps) of launch i (lwb_conv_plan_launch_info): the kernel instance is
        (n_tile, mode); k_stages = K stages of 64 per filter tap."""
        out = (ctypes.c_int * 4)()
        check(lib().lwb_conv_plan_launch_info(self._h, i, out), "lwb_conv_plan_launch_info")
        return dict(zip(("n_tile", "mode", "k_stages", "taps"), out))

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


# (N tile, operand mode) of the k_conv_wg instances ImpersonatorGenerator.inference launches by default (fp16f8): the
# row-K stem (fp16x3, swapped 64-channel tiles), every 128-wide N tile, the 128 -> 64 skipper, the folded 7x7 heads
GENERATOR_CONV_INSTANCES = ((64, 1), (128, 2), (64, 2), (32, 2))
# the HBM-bound kernels that run beside them on the other sub-batch stream: name -> (lwb_glue_kernel_resources which, c)
GENERATOR_GLUE_INSTANCES = {"k_norm_act": (0, 0), "k_norm_act<WARP> c=128": (1, 128), "k_norm_act<WARP> c=256": (1, 256),
                            "k_norm_act<WARP> c=512": (1, 512), "k_heads": (3, 0), "k_nchw_to_nhwc_split": (4, 0)}
_RES_KEYS = ("regs", "static_smem", "dyn_smem", "local_bytes", "threads", "blocks_alone", "consumer_regs")


def conv_kernel_resources(n_tile, mode):
    """Registers, shared memory and CTAs per SM of one k_conv_wg instance as launched (lwb_conv_kernel_resources)."""
    out = (ctypes.c_int * 7)()
    check(lib().lwb_conv_kernel_resources(n_tile, mode, out), "lwb_conv_kernel_resources")
    return dict(zip(_RES_KEYS, out))


def glue_kernel_resources(which, c=0):
    """The same for k_norm_act (which 0 / 1 = WARP at c channels / 2 = EXT), k_heads (3), k_nchw_to_nhwc_split (4)."""
    out = (ctypes.c_int * 6)()
    check(lib().lwb_glue_kernel_resources(which, c, out), "lwb_glue_kernel_resources")
    return dict(zip(_RES_KEYS, out))


def blocks_beside(conv, other, props):
    """Blocks of ``other`` that fit on an SM that already holds one CTA of ``conv`` (dicts of *_kernel_resources;
    ``props`` = torch.cuda.get_device_properties).  The rules of the CUDA occupancy calculator (cuda_occupancy.h):
    registers are allocated per warp in units of 256 from the register file of the warp's sub-partition (four per SM,
    warp w of a block on sub-partition w % 4), shared memory per block plus 1 KB reserved by the system."""
    def warp_regs(r):
        return -(-r * 32 // 256) * 256
    parts = 4
    per_part = props.regs_per_multiprocessor // parts
    conv_warps = conv["threads"] // 32
    used = [warp_regs(conv["regs"]) * len(range(p, conv_warps, parts)) for p in range(parts)]
    warps = other["threads"] // 32
    need = -(-warps // parts) * warp_regs(other["regs"])            # on the sub-partition that gets the most of its warps
    by_regs = min((per_part - u) // need for u in used)
    smem = lambda k: k["static_smem"] + k["dyn_smem"] + 1024
    by_smem = (props.shared_memory_per_multiprocessor - smem(conv)) // smem(other)
    by_threads = (props.max_threads_per_multi_processor - conv["threads"]) // other["threads"]
    return max(0, min(by_regs, by_smem, by_threads))


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


_staging = {}              # (device index, slot) -> (pinned uint8 buffer, event recorded after its last H2D copy)


def upload_u8(frames, device=None, slot=0):
    """A host uint8 array / tensor -> the same uint8 tensor on ``device`` (default: the current one), copied on the current
    stream through a pinned staging buffer that is reused from call to call (per device and ``slot``: a caller that keeps
    two uploads in flight uses two slots).  Waits only for the previous copy out of the same buffer."""
    a = frames.numpy() if torch.is_tensor(frames) else np.asarray(frames)
    if a.dtype != np.uint8:
        raise LwbError("frames must be uint8, got %s" % a.dtype)
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    key = (device.index, slot)
    buf, done = _staging.get(key, (None, None))
    if done is not None:
        done.synchronize()
    if buf is None or buf.numel() < a.size:
        buf = torch.empty(max(a.size, 1), dtype=torch.uint8, pin_memory=True)
    np.copyto(buf.numpy()[:a.size].reshape(a.shape), a)
    out = torch.empty(a.shape, dtype=torch.uint8, device=device)
    out.view(-1).copy_(buf[:a.size], non_blocking=True)
    done = torch.cuda.Event()
    done.record(torch.cuda.current_stream(device))
    _staging[key] = (buf, done)
    return out


def frames_in(frames, size, hmr_size=224, bgr=True, want_img=True, want_hmr=True, want_u8=False):
    """uint8 frames [n,H,W,3] or [H,W,3] (a CUDA tensor, or a host array / tensor, uploaded with ``upload_u8``), B,G,R
    as cv2.imread returns them (``bgr=False``: R,G,B) -> (img, hmr, u8), each None unless asked for:

      img  fp32 [n,3,size,size] RGB in [-1,1]: cv2.resize(rgb, (size, size)) / 255.0 * 2 - 1.0 (utils/cv_utils.py:10-47)
      hmr  fp32 [n,3,hmr_size,hmr_size] RGB in [-1,1]: the same from the frame itself (the HMR input)
      u8   uint8 [n,size,size,3] BGR: what cv_utils.save_cv2_img(frame, image_size=size) writes

    One kernel launch (lwb_frames_in); every byte equals cv2.resize's uint8 INTER_LINEAR result on the same frame."""
    if not torch.is_tensor(frames) or not frames.is_cuda:
        frames = upload_u8(frames)
    _chk_cuda(frames)
    if frames.dim() == 3:
        frames = frames[None]
    if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
        raise LwbError("frames must be uint8 [n,H,W,3] or [H,W,3], got %s %s"
                       % (str(frames.dtype).replace("torch.", ""), list(frames.shape)))
    n, h, w, _ = frames.shape
    dev = frames.device
    img = torch.empty((n, 3, size, size), dtype=torch.float32, device=dev) if want_img else None
    hmr = torch.empty((n, 3, hmr_size, hmr_size), dtype=torch.float32, device=dev) if want_hmr else None
    u8 = torch.empty((n, size, size, 3), dtype=torch.uint8, device=dev) if want_u8 else None
    _count(1)
    check(lib().lwb_frames_in(ptr(frames), n, h, w, int(bool(bgr)), size, ptr(img), hmr_size, ptr(hmr), ptr(u8), stream()),
          "lwb_frames_in")
    return img, hmr, u8


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
    if y_lo is not None and y_hi is not None and y_lo.shape != y_hi.shape:
        raise LwbError("gated_act: y_lo is %s, y_hi is %s" % (tuple(y_lo.shape), tuple(y_hi.shape)))
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
    if tuple(x.shape[:3]) != (n, h, w):
        raise LwbError("self_attention: x is %s, qkv has [n, h, w] = %s" % (tuple(x.shape), (n, h, w)))
    if tuple(bias.shape) != (2 * int(dq) + dv,):
        raise LwbError("self_attention: bias must be [%d], got %s" % (2 * int(dq) + dv, tuple(bias.shape)))
    if out is None:
        out = torch.empty_like(x)
    elif out.shape != x.shape:
        raise LwbError("self_attention: out must be %s, got %s" % (tuple(x.shape), tuple(out.shape)))
    _count(1)
    check(lib().lwb_self_attention_nhwc(ptr(qkv), ld, ptr(bias), n, h * w, int(dq), dv, ptr(x), ptr(gamma), ptr(out), stream()),
          "lwb_self_attention_nhwc")
    return out


def _ceil_pool_out(size, k, stride):
    """torch's ceil_mode output size without padding: a last window that would start past the input is dropped."""
    o = -(-(size - k) // stride) + 1
    return o - 1 if (o - 1) * stride >= size else o


def maxpool_nchw_to_nhwc(x, k, stride, out=None):
    """F.max_pool2d(x, k, stride, ceil_mode=True) (networks/hmr.py:150): NCHW fp32 -> NHWC fp32."""
    _chk_cuda(x, out)
    n, c, h, w = x.shape
    ho, wo = _ceil_pool_out(h, k, stride), _ceil_pool_out(w, k, stride)
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
    ws = _workspace(lib().lwb_smpl_workspace_bytes(B), dev, "smpl")
    check(lib().lwb_smpl_forward(
        ptr(beta), ptr(theta), B, nb, V, ptr(model["v_template"]), ptr(model["shapedirs"]), ptr(model["posedirs"]),
        ptr(model["j_template"]), ptr(model["j_shapedirs"]), ptr(model["parents"]), ptr(model["weights"]),
        ptr(model["joint_regressor_t"]), nj, 1 if rotate_base else 0,
        ptr(verts), ptr(joints), ptr(Rs), ptr(Jt), ptr(cam if j2d is not None else None), ptr(j2d), ptr(ws), stream()),
        "lwb_smpl_forward")
    _count(3 if want_joints else 2)
    return verts, joints, Rs, Jt, j2d


# ---- Mask R-CNN person detector (impersonator_b200.detectors) ------------------------------------------------------
def _i32_ptrs(values):
    """Host list of ints -> a C int array for the launchers' host-side const int* arguments."""
    return (ctypes.c_int * len(values))(*[int(v) for v in values])


def det_transform(img, ho, wo, hp, wp, out=None):
    """[3,h,w] in [-1,1] -> (img + 1) / 2, normalised, bilinear to [ho, wo], zero padded to [1,3,hp,wp]."""
    _chk_cuda(img, out)
    _, h, w = img.shape
    if out is None:
        out = torch.empty((1, 3, hp, wp), dtype=torch.float32, device=img.device)
    _count(1)
    check(lib().lwb_det_transform(ptr(img), h, w, ho, wo, hp, wp, ptr(out), stream()), "lwb_det_transform")
    return out


def det_stem_pool(x, scale, shift, y_hi, y_lo):
    _chk_cuda(x, scale, shift, y_hi, y_lo)
    n, c, h, w = x.shape
    _count(1)
    check(lib().lwb_det_stem_pool(ptr(x), n, c, h, w, ptr(scale), ptr(shift), ptr(y_hi), ptr(y_lo), stream()), "lwb_det_stem_pool")


def det_bias_act(raw, bias=None, relu=False, raw2=None, res=None, res_half=False, step=1, out_hw=None, c=None,
                 y_f32=None, y_hi=None, y_lo=None):
    """y = act(raw[step * (y, x)] + raw2 + bias + res) (res nearest-2x upsampled when res_half) -> fp32 / operands."""
    _chk_cuda(raw, raw2, bias, res, y_f32, y_hi, y_lo)
    n, h_in, w_in, ld = raw.shape
    c = c or ld
    h, w = out_hw or (h_in, w_in)
    _count(1)
    with _Prof("det", 0.0):
        check(lib().lwb_det_bias_act(ptr(raw), ld, ptr(raw2), ptr(bias), ptr(res), 1 if (res_half and res is not None) else 0, int(step), h_in, w_in,
                                     1 if relu else 0, n, h, w, c, ptr(y_f32), ptr(y_hi), ptr(y_lo), stream()), "lwb_det_bias_act")


def det_d2s_bias_relu(raw, bias, y_f32=None, y_hi=None, y_lo=None):
    _chk_cuda(raw, bias, y_f32, y_hi, y_lo)
    n, h, w, c4 = raw.shape
    _count(1)
    check(lib().lwb_det_d2s_bias_relu(ptr(raw), ptr(bias), n, h, w, c4 // 4, ptr(y_f32), ptr(y_hi), ptr(y_lo), stream()),
          "lwb_det_d2s_bias_relu")


def det_rpn(heads, strides, cell_anchors, bias, k, clip_hw, min_size, xform_clip, out):
    """heads: list of [gh,gw,16] raw head outputs; out: dict of candidate buffers (boxes, scores, groups, valid, top)."""
    _chk_cuda(bias, *heads)
    L = len(heads)
    offs, o = [], 0
    for hd in heads:
        offs.append(o)
        o += min(k, hd.shape[0] * hd.shape[1] * 3)
    hp = (ctypes.c_void_p * L)(*[h.data_ptr() for h in heads])
    cell = cell_anchors.detach().cpu().float().contiguous().numpy()
    cell_c = (ctypes.c_float * cell.size)(*cell.ravel().tolist())
    _count(1)
    check(lib().lwb_det_rpn(L, hp, _i32_ptrs([h.shape[0] for h in heads]), _i32_ptrs([h.shape[1] for h in heads]),
                            _i32_ptrs([s[0] for s in strides]), _i32_ptrs([s[1] for s in strides]), cell_c,
                            _i32_ptrs(offs), ptr(bias), int(k), float(clip_hw[0]), float(clip_hw[1]), float(min_size),
                            float(xform_clip), ptr(out.get("top")), ptr(out["boxes"]), ptr(out["scores"]), ptr(out["groups"]),
                            ptr(out["valid"]), stream()), "lwb_det_rpn")
    return o


def det_nms(boxes, scores, groups, valid, thresh, max_keep, m_max=None, out=None):
    """Batched NMS (per group, torchvision's vanilla branch) over n slots -> dict(keep, boxes, scores, groups, count)."""
    _chk_cuda(boxes, scores, groups, valid)
    n = scores.shape[0]
    m_max = m_max or n
    dev = scores.device
    if out is None:
        out = dict(keep=torch.empty(max_keep, dtype=torch.int32, device=dev), boxes=torch.empty((max_keep, 4), dtype=torch.float32, device=dev),
                   scores=torch.empty(max_keep, dtype=torch.float32, device=dev), groups=torch.empty(max_keep, dtype=torch.int32, device=dev),
                   count=torch.empty(1, dtype=torch.int32, device=dev))
    ws = _workspace(lib().lwb_det_nms_workspace_bytes(n, m_max), dev, "nms")
    _count(4)
    with _Prof("det", 0.0, "nms"):
        check(lib().lwb_det_nms(ptr(boxes), ptr(scores), ptr(groups), ptr(valid), n, int(m_max), float(thresh), int(max_keep), ptr(ws),
                                ptr(out["keep"]), ptr(out["boxes"]), ptr(out["scores"]), ptr(out["groups"]), ptr(out["count"]), stream()),
              "lwb_det_nms")
    return out


def det_roi_align(feats, boxes, count, out_size, sampling=2, levels=None, y_f32=None, y_hi=None, y_lo=None):
    """MultiScaleRoIAlign over 4 NHWC fp32 levels [1,h,w,c] -> RoI-major [r_max,out,out,c]."""
    _chk_cuda(boxes, count, levels, y_f32, y_hi, y_lo, *feats)
    c = feats[0].shape[-1]
    fp = (ctypes.c_void_p * 4)(*[f.data_ptr() for f in feats])
    _count(1)
    with _Prof("det", 0.0, "roi_align"):
        check(lib().lwb_det_roi_align(fp, _i32_ptrs([f.shape[1] for f in feats]), _i32_ptrs([f.shape[2] for f in feats]), c,
                                      ptr(boxes), ptr(count), boxes.shape[0], int(out_size), int(sampling), ptr(levels),
                                      ptr(y_f32), ptr(y_hi), ptr(y_lo), stream()), "lwb_det_roi_align")


def det_box_candidates(pred, nc, proposals, count, clip_hw, score_thresh, min_size, xform_clip, out):
    _chk_cuda(pred, proposals, count)
    r_max, ld = pred.shape
    _count(1)
    check(lib().lwb_det_box_candidates(ptr(pred), ld, int(nc), ptr(proposals), ptr(count), r_max, float(clip_hw[0]), float(clip_hw[1]),
                                       float(score_thresh), float(min_size), float(xform_clip), ptr(out["boxes"]), ptr(out["scores"]),
                                       ptr(out["groups"]), ptr(out["valid"]), stream()), "lwb_det_box_candidates")


def det_mask_probs(raw, bias, labels, count, logits=None, probs=None):
    _chk_cuda(raw, bias, labels, count, logits, probs)
    d_max, h, w, ld = raw.shape
    _count(1)
    check(lib().lwb_det_mask_probs(ptr(raw), ld, ptr(bias), ptr(labels), ptr(count), d_max, h * w, ptr(logits), ptr(probs), stream()),
          "lwb_det_mask_probs")


def det_paste_masks(probs, boxes, count, ratio_hw, hw, masks=None, out_boxes=None):
    """resize_boxes + paste_masks_in_image: probs [d,m,m], boxes [d,4] -> masks [d,1,h,w] (None: boxes only), boxes [d,4]."""
    _chk_cuda(probs, boxes, count, masks, out_boxes)
    d_max, m = probs.shape[0], probs.shape[-1]
    _count(1)
    check(lib().lwb_det_paste_masks(ptr(probs), m, ptr(boxes), ptr(count), d_max, float(ratio_hw[0]), float(ratio_hw[1]),
                                    int(hw[0]), int(hw[1]), ptr(masks), ptr(out_boxes), stream()), "lwb_det_paste_masks")


def det_person_mask(boxes, labels, count, masks, thresh, ks, person=1):
    """-> (pid int32[1], box [4], dilated {0,1} mask [1,1,h,w]) of the largest-area person (the last detection if none)."""
    _chk_cuda(boxes, labels, count, masks)
    h, w = masks.shape[-2:]
    dev = masks.device
    pid = torch.empty(1, dtype=torch.int32, device=dev)
    box = torch.empty(4, dtype=torch.float32, device=dev)
    out = torch.empty((1, 1, h, w), dtype=torch.float32, device=dev)
    _count(1)
    check(lib().lwb_det_person_mask(ptr(boxes), ptr(labels), ptr(count), int(person), ptr(masks), h, w, float(thresh), int(ks),
                                    ptr(pid), ptr(box), ptr(out), stream()), "lwb_det_person_mask")
    return pid, box, out


# ---- paired image-quality metrics (impersonator_b200.metrics) -----------------------------------------------------
def conv2d_direct_relu_nhwc(x, w, bias=None, stride=1, pad=0, out=None):
    """relu(conv2d(x, w, bias, stride, pad)): x NCHW fp32 -> NHWC fp32 [n,ho,wo,cout]."""
    _chk_cuda(x, w, bias, out)
    n, cin, h, wd = x.shape
    cout, _, kh, kw = w.shape
    ho, wo = (h + 2 * pad - kh) // stride + 1, (wd + 2 * pad - kw) // stride + 1
    if out is None:
        out = torch.empty((n, ho, wo, cout), dtype=torch.float32, device=x.device)
    _count(1)
    check(lib().lwb_conv2d_direct_relu_nhwc(ptr(x), ptr(w), ptr(bias), n, cin, h, wd, cout, kh, kw, stride, pad, ptr(out),
                                            stream()), "lwb_conv2d_direct_relu_nhwc")
    return out


def maxpool_nhwc(x, k, stride, y_f32=None, y_hi=None, y_lo=None):
    """F.max_pool2d(x, k, stride) (floor mode) on NHWC fp32 -> y_f32 and / or fp16 hi / lo operands; with no output
    given, a new fp32 tensor is returned."""
    _chk_cuda(x, y_f32, y_hi, y_lo)
    n, h, w, c = x.shape
    if y_f32 is None and y_hi is None:
        y_f32 = torch.empty((n, (h - k) // stride + 1, (w - k) // stride + 1, c), dtype=torch.float32, device=x.device)
    _count(1)
    check(lib().lwb_maxpool_nhwc(ptr(x), n, h, w, c, k, stride, ptr(y_f32), ptr(y_hi), ptr(y_lo), stream()), "lwb_maxpool_nhwc")
    return y_f32


def _chk_frames(*ts):
    _chk_cuda(*ts)
    shape = ts[0].shape
    for t in ts:
        if t.dtype != torch.float32 or t.dim() != 4 or t.shape[1] != 3 or t.shape != shape:
            raise LwbError("frames must be float32 [n,3,h,w] of one shape, got %s / %s" % (tuple(shape), tuple(t.shape)))


def ssim_psnr(pred, ref, from01=False, ssim=None, psnr=None):
    """Per-frame SSIM and PSNR (lwb_ssim_psnr) of [n,3,h,w] fp32 frames in [-1,1] ([0,1] with from01) -> fp64 [n], [n]."""
    _chk_frames(pred, ref)
    n, _, h, w = pred.shape
    dev = pred.device
    if ssim is None:
        ssim = torch.empty(n, dtype=torch.float64, device=dev)
        psnr = torch.empty(n, dtype=torch.float64, device=dev)
    ws = _workspace(lib().lwb_ssim_psnr_workspace_bytes(n, h, w), dev, "ssim")
    _count(2)
    with _Prof("metrics", 0.0, "ssim_psnr"):
        check(lib().lwb_ssim_psnr(ptr(pred), ptr(ref), n, h, w, 1 if from01 else 0, ptr(ws), ptr(ssim), ptr(psnr), stream()),
              "lwb_ssim_psnr")
    return ssim, psnr


def lpips_input(pred, ref, from01=False, out=None):
    """PNetLin's scaling layer of pred and ref as one batch [2n,3,h,w] (pred first)."""
    _chk_frames(pred, ref)
    n, _, h, w = pred.shape
    if out is None:
        out = torch.empty((2 * n, 3, h, w), dtype=torch.float32, device=pred.device)
    _chk_cuda(out)
    _count(1)
    check(lib().lwb_lpips_input(ptr(pred), ptr(ref), n, h, w, 1 if from01 else 0, ptr(out), stream()), "lwb_lpips_input")
    return out


def lpips_layer(feat, lin, layer, layers, score):
    """One LPIPS tap of feat NHWC [2n,h,w,c] into layers [n, L] (column ``layer``) and score [n] (= for layer 0, += after)."""
    _chk_cuda(feat, lin, layers, score)
    n2, h, w, c = feat.shape
    if lin.numel() != c or layers.dim() != 2 or layers.shape[0] != n2 // 2 or score.numel() != n2 // 2:
        raise LwbError("lpips_layer: %d channels, %d lin weights, layers %s, score %s" % (c, lin.numel(), tuple(layers.shape),
                                                                                           tuple(score.shape)))
    _count(1)
    check(lib().lwb_lpips_layer(ptr(feat), n2 // 2, h * w, c, ptr(lin), int(layer), layers.shape[1], ptr(layers), ptr(score),
                                stream()), "lwb_lpips_layer")


# ---- unpaired image-quality metrics: InceptionV3 features (impersonator_b200.metrics) ------------------------------
def inception_input(x, out=None):
    """[n,3,h,w] fp32 frames in [0,1] -> x * 2 - 1 bilinearly resized to [n,3,299,299] (align_corners=False)."""
    _chk_frames(x)
    n, _, h, w = x.shape
    if out is None:
        out = torch.empty((n, 3, 299, 299), dtype=torch.float32, device=x.device)
    _chk_cuda(out)
    if tuple(out.shape) != (n, 3, 299, 299):
        raise LwbError("inception_input: out must be [%d,3,299,299], got %s" % (n, tuple(out.shape)))
    _count(1)
    check(lib().lwb_inception_input(ptr(x), n, h, w, ptr(out), stream()), "lwb_inception_input")
    return out


def bn_act_segment(raw, c0, c, scale=None, shift=None, relu=True, box=False, c_out=None, y_f32=None, y_hi=None, y_lo=None,
                   off_y=0):
    """relu?(r * scale + shift) of channels [c0, c0+c) of raw NHWC fp32 [n,h,w,ld] (r = their 3x3 box mean / 9 with
    ``box``) -> channels [off_y, off_y + c_out) of y_f32 and / or fp16 y_hi / y_lo (one pitch, channels >= c zero)."""
    _chk_cuda(raw, scale, shift, y_f32, y_hi, y_lo)
    n, h, w, ld = raw.shape
    c_out = c_out or c
    ys = [t for t in (y_f32, y_hi, y_lo) if t is not None]
    if not ys or any(t.shape[:3] != raw.shape[:3] or t.shape[3] != ys[0].shape[3] for t in ys):
        raise LwbError("bn_act_segment: outputs must be [%d,%d,%d,pitch] of one pitch" % (n, h, w))
    if scale is not None and (scale.numel() != c or shift.numel() != c):
        raise LwbError("bn_act_segment: scale / shift must hold %d values" % c)
    _count(1)
    check(lib().lwb_bn_act_segment(ptr(raw), n, h, w, ld, int(c0), int(c), int(c_out), 1 if box else 0, ptr(scale), ptr(shift),
                                   1 if relu else 0, ptr(y_f32), ptr(y_hi), ptr(y_lo), ys[0].shape[3], int(off_y), stream()),
          "lwb_bn_act_segment")


def maxpool_nhwc_slice(x, c, k, stride, y_f32=None, y_hi=None, y_lo=None, off_y=0):
    """F.max_pool2d(x[..., :c], k, stride) (floor mode) of NHWC fp32 x -> channels [off_y, off_y + c) of the outputs."""
    _chk_cuda(x, y_f32, y_hi, y_lo)
    n, h, w, ld_x = x.shape
    ys = [t for t in (y_f32, y_hi, y_lo) if t is not None]
    ho, wo = (h - k) // stride + 1, (w - k) // stride + 1
    if not ys or any(tuple(t.shape[:3]) != (n, ho, wo) or t.shape[3] != ys[0].shape[3] for t in ys):
        raise LwbError("maxpool_nhwc_slice: outputs must be [%d,%d,%d,pitch] of one pitch" % (n, ho, wo))
    _count(1)
    check(lib().lwb_maxpool_nhwc_slice(ptr(x), n, h, w, int(c), ld_x, k, stride, ptr(y_f32), ptr(y_hi), ptr(y_lo),
                                       ys[0].shape[3], int(off_y), stream()), "lwb_maxpool_nhwc_slice")
