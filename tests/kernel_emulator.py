"""TEST INFRASTRUCTURE ONLY -- torch-CPU stand-ins for the C-ABI front-ends of impersonator_b200.kernels.

The host mirrors (generator / hmr / inpaintor / LPIPS / Inception streams) are pure orchestration: they bind buffers,
fold BatchNorms, stack gated filters, fold the 7x7 heads into a 7x1 filter, chain conv plans and epilogues.  None of that needs a GPU to be
wrong.  ``install(monkeypatch)`` replaces every kernel front-end the streams call by a plain torch implementation of the
SAME contract (include/lwb_b200.h), so the CPU suite can run the whole host logic against the oracles.  The emulation
works on the fp16 hi/lo operand pairs (run it with LWB_PRECISION=fp16x3); it is never used by the product.
"""
import numpy as np
import torch
import torch.nn.functional as F

from conv_emulation import act_pair_blocks, fp16_pair, range_bits
from frames_in_cases import cv2_route
from impersonator_b200 import kernels as K
from impersonator_b200.binding import RANGE_HEADS


def _pair_to_f32(pair):
    hi, lo = pair
    return hi.float() + (lo.float() if lo is not None else 0.0)


def _emit(y, y_hi, y_lo, lo_format, range_flag):
    """y [..., c] -> the operands y_hi / y_lo (nullable) [..., c_pad >= c], channels >= c zero, and the range bits."""
    v = torch.zeros(y_hi.shape)
    v[..., :y.shape[-1]] = y
    hi, lo = fp16_pair(v)
    y_hi.copy_(hi)
    if y_lo is not None and lo_format == 1:
        y_lo.view(torch.uint8).copy_(act_pair_blocks(v, hi))
    elif y_lo is not None:
        y_lo.copy_(lo)
    if range_flag is not None:
        range_flag |= range_bits(hi)


class PackedWeight(tuple):
    pass


def pack_conv_weight(w, transposed=False, cout_pad=None, cin_pad=None, split=True, absmax=None):
    w = w.detach().float()
    if transposed:
        cin, cout = w.shape[:2]
    else:
        cout, cin = w.shape[:2]
    cout_pad, cin_pad = cout_pad or cout, cin_pad or cin
    full = torch.zeros((cin_pad, cout_pad) + tuple(w.shape[2:])) if transposed else torch.zeros((cout_pad, cin_pad) + tuple(w.shape[2:]))
    if transposed:
        full[:cin, :cout] = w
    else:
        full[:cout, :cin] = w
    pw = PackedWeight((full, transposed))
    pw.w_exp = 15
    return pw


def pack_conv_weight_rowk(w, cout_pad=None, cpx=8, kxs=8, split=True, absmax=None):
    pw = PackedWeight((w.detach().float(), "rowk"))
    pw.w_exp = 15
    return pw


class ConvPlan(object):
    """lwb_conv_plan_create / run on NHWC hi/lo pairs -> raw fp32 NHWC (+ InstanceNorm sums in f64)."""

    def __init__(self, desc, x0, x1, w, out_raw, stats):
        self.desc, self.x0, self.x1, self.w, self.out, self.stats = desc, x0, x1, w, out_raw, stats
        self.num_launches = 1
        self.flops = 0.0
        self.label = "emulated"
        self.prof_class = "conv"

    def run(self):
        d = self.desc
        x = _pair_to_f32(self.x0)
        if self.x1 is not None:
            x = torch.cat([x, _pair_to_f32(self.x1)], dim=-1)
        w, kind = self.w
        if kind == "rowk":
            # padded NHWC8 input [n, h+6, w+8, 8] holding pixel (y,x) at (y+3, x+3); 7x7 stride 1
            x = x[:, :, :d.w_in + 6, :w.shape[1]].permute(0, 3, 1, 2)
            y = F.conv2d(x, w)
        else:
            x = x.permute(0, 3, 1, 2)
            if d.transposed == 2:
                # merged transposed conv (lwb_conv_desc.transposed = 2): weights [4*cout, cin, 2, 2], tap (dy, dx) reads
                # in[y+dy, x+dx] (zero beyond the border), column block 2a+b is output pixel (2y+a, 2x+b)
                y4 = F.conv2d(F.pad(x, (0, 1, 0, 1)), w)
                n_, c4, h_, w_ = y4.shape
                y = y4.view(n_, 2, 2, c4 // 4, h_, w_).permute(0, 3, 4, 1, 5, 2).reshape(n_, c4 // 4, 2 * h_, 2 * w_)
            elif kind:
                y = F.conv_transpose2d(x, w, stride=2, padding=1, output_padding=1)
            else:
                pw = d.pad_w if d.pad_w >= 0 else d.pad
                y = F.conv2d(x, w, stride=d.stride, padding=(d.pad, pw), dilation=d.dil)
        y = y.permute(0, 2, 3, 1)
        assert tuple(y.shape) == tuple(self.out.shape), (tuple(y.shape), tuple(self.out.shape))
        self.out.copy_(y)
        if self.stats is not None:
            self.stats[..., 0] += y.double().sum(dim=(1, 2))
            self.stats[..., 1] += (y.double() ** 2).sum(dim=(1, 2))


def _warp(src, T, h, w, align_corners):
    Ts = F.interpolate(T.permute(0, 3, 1, 2), size=(h, w), mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
    x = src.permute(0, 3, 1, 2)
    if x.shape[0] != T.shape[0]:
        x = x.expand(T.shape[0], -1, -1, -1)
    return F.grid_sample(x, Ts, mode='bilinear', padding_mode='zeros', align_corners=bool(align_corners)).permute(0, 2, 3, 1)


def norm_act_nhwc(raw, stats, gamma, beta, relu, ws, eps=1e-5, residual=None, warp_src=None, T=None, align_corners=False,
                  y_f32=None, y_hi=None, y_lo=None, lo_format=0, post_scale=None, post_shift=None, post_relu=False,
                  res_step=1, range_flag=None):
    n, h, w, c = raw.shape
    v = raw.double()
    if stats is not None:
        mean = stats[..., 0] / (h * w)
        var = (stats[..., 1] / (h * w) - mean * mean).clamp(min=0)
        scale = (gamma.double() if gamma is not None else 1.0) / torch.sqrt(var + eps)
        shift = (beta.double() if beta is not None else 0.0) - mean * scale
        v = v * scale[:, None, None, :] + shift[:, None, None, :]
    elif gamma is not None or beta is not None:
        v = v * (gamma.double() if gamma is not None else 1.0) + (beta.double() if beta is not None else 0.0)
    v = v.float()
    if relu:
        v = F.relu(v)
    if residual is not None:
        v = v + residual[:, ::res_step, ::res_step, :]
    if warp_src is not None:
        v = v + _warp(warp_src, T, h, w, align_corners)
    ops = v
    if post_scale is not None:
        ops = v * post_scale + post_shift
        if post_relu:
            ops = F.relu(ops)
    if y_f32 is not None:
        y_f32.copy_(v)
    if y_hi is not None:
        _emit(ops, y_hi, y_lo, lo_format, range_flag)


def nchw_to_nhwc_split(x, c_pad=None, pad_hw=(0, 0, 0, 0), hi=None, lo=None, split=True):
    n, c, h, w = x.shape
    c_pad = c_pad or c
    top, bottom, left, right = pad_hw
    full = torch.zeros((n, h + top + bottom, w + left + right, c_pad))
    full[:, top:top + h, left:left + w, :c] = x.permute(0, 2, 3, 1)
    if hi is None:
        hi = torch.empty(full.shape, dtype=torch.float16)
        lo = torch.empty_like(hi) if split else None
    h, l = fp16_pair(full)
    hi.copy_(h)
    if lo is not None:
        lo.copy_(l)
    return hi, lo


def nhwc_to_nchw(x, c=None, out=None):
    c = c or x.shape[3]
    y = x[..., :c].permute(0, 3, 1, 2).contiguous()
    if out is not None:
        out.copy_(y)
        return out
    return y


def conv2d_direct_nchw(x, w, bias=None, stride=1, pad=0, dil=1):
    return F.conv2d(x, w, bias, stride=stride, padding=pad, dilation=dil)


def gated_bn_nchw(ab, act, scale=None, shift=None):
    c = ab.shape[1] // 2
    a, g = ab[:, :c], ab[:, c:]
    a = F.leaky_relu(a, 0.2) if act == 2 else (F.relu(a) if act == 1 else a)
    y = a * torch.sigmoid(g)
    if scale is not None:
        y = y * scale[None, :, None, None] + shift[None, :, None, None]
    return y


def gated_act_nhwc(raw, c, bias, act, scale, shift, upsample=1, clamp=False, y_f32=None, y_hi=None, y_lo=None,
                   lo_format=0, range_flag=None):
    a, g = raw[..., :c], raw[..., c:2 * c]
    if bias is not None:
        a, g = a + bias[:c], g + bias[c:]
    a = F.leaky_relu(a, 0.2) if act == 2 else a
    y = a * torch.sigmoid(g)
    if scale is not None:
        y = y * scale + shift
    if clamp:
        y = y.clamp(-1, 1)
    if upsample == 2:
        y = y.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    if y_f32 is not None:
        y_f32[..., :c] = y                          # columns c.. of a wider f32 buffer are left alone
    if y_hi is not None:
        _emit(y, y_hi, y_lo, lo_format, range_flag)


def self_attention_nhwc(qkv, bias, x, gamma, dq=16, out=None):
    n, h, w, ld = qkv.shape
    dv = x.shape[3]
    t = (qkv[..., :2 * dq + dv] + bias).view(n, h * w, 2 * dq + dv)
    q, k, v = t[..., :dq], t[..., dq:2 * dq], t[..., 2 * dq:]
    att = torch.softmax(torch.bmm(q, k.transpose(1, 2)), dim=-1)
    y = (gamma * torch.bmm(att, v) + x.view(n, h * w, dv)).view(n, h, w, dv)
    if out is not None:
        out.copy_(y)
        return out
    return y


def maxpool_nchw_to_nhwc(x, k, stride, out=None):
    y = F.max_pool2d(x, kernel_size=k, stride=stride, ceil_mode=True).permute(0, 2, 3, 1).contiguous()
    if out is not None:
        out.copy_(y)
        return out
    return y


def global_avgpool_nhwc(x, scale=None, shift=None, relu=False, out=None, ld_out=None):
    v = x
    if scale is not None:
        v = v * scale + shift
    if relu:
        v = F.relu(v)
    y = v.mean(dim=(1, 2))
    if out is None:
        return y
    out[:, :y.shape[1]] = y
    return out


def linear(x, w, bias=None, relu=False, out=None, accumulate=False):
    y = F.linear(x, w, bias)
    if relu:
        y = F.relu(y)
    if out is None:
        return y
    if accumulate:
        out += y
    else:
        out.copy_(y)
    return out


def pack_head_weights(w_img, w_att):
    return torch.cat([w_img, w_att], dim=0).float()


def conv7x7_heads_nhwc(x, w4, out=None):
    y = F.conv2d(x.permute(0, 3, 1, 2), w4, padding=3).permute(0, 2, 3, 1)
    if out is not None:
        out.copy_(y)
        return out
    return y


def heads_composite(raw, bg=None, want_color=True, want_mask=True, color=None, mask=None, pred=None, want_pred=True,
                    pred_hwc=None, pred_u8=None, folded_kw=0, range_flag=None):
    n, h, w, cs = raw.shape
    if folded_kw:
        r = torch.zeros(n, h, w, 4)
        for kx in range(folded_kw):
            sh = kx - folded_kw // 2                       # out[y, x] += raw[y, x + sh, kx*4 : kx*4+4]
            x0, x1 = max(0, -sh), min(w, w - sh)           # (no column inside the image when w <= |sh|)
            if x1 > x0:
                r[:, :, x0:x1] += raw[:, :, x0 + sh:x1 + sh, kx * 4:kx * 4 + 4]
    else:
        r = raw[..., :4]
    col = torch.tanh(r[..., :3]).permute(0, 3, 1, 2)
    m = torch.sigmoid(r[..., 3:4]).permute(0, 3, 1, 2)
    p = None
    if bg is not None:
        p = m * bg + (1 - m) * col
    outs = []
    for given, val in ((color, col), (mask, m), (pred, p)):
        if given is not None and val is not None:
            given.copy_(val)
            outs.append(given)
        else:
            outs.append(val.contiguous() if val is not None else None)
    if pred_hwc is not None:
        pred_hwc.copy_(p.permute(0, 2, 3, 1))
    if pred_u8 is not None:                                  # float32 ((img + 1) / 2.0 * 255) truncated, BGR
        pred_u8.copy_(((p.permute(0, 2, 3, 1) + 1) / 2.0 * 255).to(torch.uint8).flip(-1))
    if range_flag is not None and bool((~(r.abs() < 8)).any()):
        range_flag |= RANGE_HEADS                            # a pre-activation of magnitude >= 8, or NaN
    return tuple(outs)


def correspond(cam, verts, face_idx, image_size, map_fn, src_p2verts, src_img=None, align_corners=None,
               want_f2verts=False, near=K.NEAR, far=K.FAR, out=None):
    """lwb_correspond's contract through the CPU oracle (oracle/nmr_ref.py + the C rasterizer restatement): one source
    for every frame or one per frame, written into the caller's ``out`` buffers when given."""
    from oracle import nmr_ref
    ac = K.default_align_corners() if align_corners is None else align_corners
    img = src_img if src_img is not None else torch.zeros(1, 3, image_size, image_size)
    c = nmr_ref.correspond(cam, verts, face_idx, map_fn, src_p2verts, img, image_size, align_corners=ac, near=near, far=far)
    res = dict(fim=c["fim"], wim=c["wim"], T=c["T"], tsf_inputs=c["tsf_inputs"].contiguous(),
               f2verts=c["f2verts"] if want_f2verts else None)
    if out is not None:
        for k in ("fim", "wim", "T", "tsf_inputs"):
            out[k].copy_(res[k])
        if out.get("f2verts") is not None:
            out["f2verts"].copy_(c["f2verts"])
        res = out
    res["tsf_img"] = res["tsf_inputs"][:, :3]
    res["cond"] = res["tsf_inputs"][:, 3:]
    return res


def warp_nchw(x, T, align_corners=None, out=None, accumulate=False):
    ac = K.default_align_corners() if align_corners is None else align_corners
    h, w = x.shape[2:]
    if tuple(T.shape[1:3]) != (h, w):                       # the flow is resized to the image (align_corners=True)
        T = F.interpolate(T.permute(0, 3, 1, 2), size=(h, w), mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
    y = torch.nn.functional.grid_sample(x.expand(T.shape[0], -1, -1, -1), T, mode='bilinear', padding_mode='zeros',
                                        align_corners=ac)
    if out is not None:
        out.copy_(out + y if accumulate else y)
        return out
    return y


def _store(y, y_f32, y_hi, y_lo, off=0):
    """y -> channels [off, off + y.shape[-1]) of the outputs; the other channels are left alone."""
    c = y.shape[-1]
    if y_f32 is not None:
        y_f32[..., off:off + c] = y
    if y_hi is not None:
        hi, lo = fp16_pair(y)
        y_hi[..., off:off + c] = hi
        if y_lo is not None:
            y_lo[..., off:off + c] = lo


def det_bias_act(raw, bias=None, relu=False, raw2=None, res=None, res_half=False, step=1, out_hw=None, c=None,
                 y_f32=None, y_hi=None, y_lo=None):
    n, h_in, w_in, ld = raw.shape
    c = c or ld
    h, w = out_hw or (h_in, w_in)
    v = raw[:, ::step, ::step, :c][:, :h, :w]
    if raw2 is not None:
        v = v + raw2[:, ::step, ::step, :c][:, :h, :w]
    if bias is not None:
        v = v + bias[:c]
    if res is not None:
        if res_half:
            v = v + res.reshape(n, h // 2, w // 2, c).repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
        else:
            v = v + res.reshape(n, h, w, c)
    if relu:
        v = F.relu(v)
    _store(v, None if y_f32 is None else y_f32.view(n, h, w, c), y_hi, y_lo)


def conv2d_direct_relu_nhwc(x, w, bias=None, stride=1, pad=0, out=None):
    y = F.relu(F.conv2d(x, w, bias, stride=stride, padding=pad)).permute(0, 2, 3, 1)
    if out is None:
        return y.contiguous()
    out.copy_(y)
    return out


def maxpool_nhwc(x, k, stride, y_f32=None, y_hi=None, y_lo=None):
    y = F.max_pool2d(x.permute(0, 3, 1, 2), k, stride).permute(0, 2, 3, 1)
    if y_f32 is None and y_hi is None:
        return y.contiguous()
    _store(y, y_f32, y_hi, y_lo)
    return y_f32


def maxpool_nhwc_slice(x, c, k, stride, y_f32=None, y_hi=None, y_lo=None, off_y=0):
    _store(F.max_pool2d(x[..., :c].permute(0, 3, 1, 2), k, stride).permute(0, 2, 3, 1), y_f32, y_hi, y_lo, off_y)


def bn_act_segment(raw, c0, c, scale=None, shift=None, relu=True, box=False, c_out=None, y_f32=None, y_hi=None, y_lo=None,
                   off_y=0):
    r = raw[..., c0:c0 + c]
    if box:
        r = F.avg_pool2d(r.permute(0, 3, 1, 2), 3, 1, 1, count_include_pad=True).permute(0, 2, 3, 1)
    v = r * scale + shift if scale is not None else r
    if relu:
        v = F.relu(v)
    _store(F.pad(v, (0, (c_out or c) - c)), y_f32, y_hi, y_lo, off_y)


_LPIPS_SHIFT, _LPIPS_SCALE = (-.030, -.088, -.188), (.458, .448, .450)


def lpips_input(pred, ref, from01=False, out=None):
    x = torch.cat([pred, ref])
    if from01:
        x = x * 2 - 1
    shift = torch.tensor(_LPIPS_SHIFT, dtype=torch.float32).view(1, 3, 1, 1)
    scale = torch.tensor(_LPIPS_SCALE, dtype=torch.float32).view(1, 3, 1, 1)
    y = (x - shift) / scale
    if out is None:
        return y
    out.copy_(y)
    return out


def lpips_layer(feat, lin, layer, layers, score):
    n = feat.shape[0] // 2
    f = feat.double()
    f = f / (f.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
    v = ((f[n:] - f[:n]) ** 2 * lin.double()).sum(-1).mean(dim=(1, 2)).float()
    layers[:, layer] = v
    score.copy_(v if layer == 0 else score + v)


def inception_input(x, out=None):
    y = F.interpolate(x * 2 - 1, size=(299, 299), mode='bilinear', align_corners=False)
    if out is None:
        return y
    out.copy_(y)
    return out


def frames_in(frames, size, hmr_size=224, bgr=True, want_img=True, want_hmr=True, want_u8=False):
    """lwb_frames_in's contract through cv2 itself (frames_in_cases.cv2_route), frame by frame, into host tensors."""
    a = frames.cpu().numpy() if torch.is_tensor(frames) else np.asarray(frames)
    routes = [cv2_route(f, size, bgr=bgr, hmr_size=hmr_size) for f in (a[None] if a.ndim == 3 else a)]
    return tuple(torch.from_numpy(np.stack([r[k] for r in routes])) if want else None
                 for k, want in enumerate((want_img, want_hmr, want_u8)))


def install_tasks(monkeypatch):
    """install() + the input-path, correspondence and warp front-ends and the renderer's CUDA-only guard: enough to run
    the task classes' personalize / view / swap on CPU (Imitator.inference itself drives CUDA streams and stays
    GPU-only)."""
    from impersonator_b200 import nmr
    install(monkeypatch)
    monkeypatch.setattr(K, "frames_in", frames_in)
    monkeypatch.setattr(K, "correspond", correspond)
    monkeypatch.setattr(K, "warp_nchw", warp_nchw)

    def _correspond(self, cam, vertices, src_p2verts, src_img, want_f2verts=False, align_corners=None):
        if src_p2verts is None:
            src_p2verts = torch.zeros((1, self.nf, 3, 2), dtype=torch.float32)
        return correspond(cam.float(), vertices.float(), self.faces, self.image_size, self.map_fn, src_p2verts.float(),
                          src_img, align_corners=align_corners, want_f2verts=want_f2verts)
    monkeypatch.setattr(nmr.SMPLRenderer, "_correspond", _correspond)


def install(monkeypatch):
    for name in ("pack_conv_weight", "pack_conv_weight_rowk", "ConvPlan", "norm_act_nhwc", "nchw_to_nhwc_split", "nhwc_to_nchw",
                 "conv2d_direct_nchw", "gated_bn_nchw", "gated_act_nhwc", "self_attention_nhwc", "maxpool_nchw_to_nhwc",
                 "global_avgpool_nhwc", "linear", "pack_head_weights", "conv7x7_heads_nhwc", "heads_composite",
                 "det_bias_act", "conv2d_direct_relu_nhwc", "maxpool_nhwc", "maxpool_nhwc_slice", "bn_act_segment",
                 "lpips_input", "lpips_layer", "inception_input"):
        monkeypatch.setattr(K, name, globals()[name])
    monkeypatch.setenv("LWB_PRECISION", "fp16x3")
