"""Host-side mirror of networks/generator.py (the reference's generator), running on the
hand-written sm_90a conv engine behind the C ABI.

Same class names, constructor arguments, method signatures and ``state_dict`` keys as the
reference, so checkpoints (``BaseModel._load_params``, models/models.py:159-179) and callers
(models/imitator.py, swapper.py, viewer.py) work unchanged:

  ResidualBlock            networks/generator.py:8-20
  ResNetGenerator          networks/generator.py:23-65     (BG net)
  ResUnetGenerator         networks/generator.py:68-184    (SID / TSF nets)
  ImpersonatorGenerator    networks/generator.py:187-320   (forward, encode_src, infer_front, swap,
                                                            inference, resize_trans, stn, transform)

The ``nn.Conv2d`` / ``nn.InstanceNorm2d`` / ``nn.ConvTranspose2d`` children are parameter holders
only (they give the reference's key names and default init); every forward path goes through
``_UnetStream`` / ``_ResnetStream`` below, which drive hand-written sm_90a kernels:
wgmma implicit-GEMM convs (fp16 hi/lo split operands, fp32 accumulate), a fused
InstanceNorm+ReLU+residual+Liquid-Warping-Block kernel, and the 7x7 heads.  There is no torch
fallback: without the CUDA library the calls raise.

Extensions over the reference (all optional): source features may have batch 1 while the target
batch is B (torch's grid_sample cannot broadcast); ``LWB_PRECISION=fp16`` selects the
single-pass "fast" mode (the default ``fp16f8`` and ``fp16x3`` both meet the 1e-3 parity bar, see binding.split_mode);
the LWB's grid_sample follows the reference's pinned torch 1.2 (align_corners=True), ``LWB_ALIGN_CORNERS=0``
selects what torch >= 1.3 does for the same flag-less call (kernels.default_align_corners).
"""
import os

import torch
import torch.nn as nn

from . import kernels as K
from ._lib import LwbError
from .binding import Operands, StreamOwner, pack_all, precision_mode, split_mode, stream_for


_WEIGHTS_EPOCH = [0]
_PASS = [0]                                              # bumped by every ImpersonatorGenerator entry point; streams stamp it


def _new_pass():
    _PASS[0] += 1



def weights_epoch():
    """Bumped whenever a network's parameters may have changed (load_state_dict, init_weights, .to()/.half()...): packed
    weights and per-shape streams are rebuilt then, and anything that cached launches against them must be rebuilt too."""
    return _WEIGHTS_EPOCH[0]


def _sub_batches(B, enc_w, res_w, bg):
    """LWB_STREAMS (default 2, at most 2): number of concurrent sub-batches ImpersonatorGenerator.inference splits a batch
    into.  Only when the source features / background are shared by the batch (the imitation case), B divides evenly and
    every sub-batch keeps at least 4 frames."""
    try:
        n = min(2, int(os.environ.get("LWB_STREAMS", "2")))
    except ValueError:
        n = 1
    if n <= 1 or B % n or B // n < 4:
        return 1
    shared = all(t is None or t.shape[0] == 1 for t in list(enc_w) + list(res_w)) and (bg is None or bg.shape[0] == 1)
    return n if shared else 1


def _tc_heads():
    """LWB_TC_HEADS (default 1): the 7x7 output heads run on the tensor cores as a 7x1 filter whose N dimension
    carries the 7 filter columns x 4 head channels (28 -> 32); the composite kernel sums the columns.  0 = the fp32
    CUDA-core kernel (k_heads7x7)."""
    return os.environ.get("LWB_TC_HEADS", "1") != "0"


def _convt_merge():
    """LWB_CONVT_MERGE (default 1): ConvTranspose2d(k3, s2, p1, op1) layers with up to 128 output channels run as ONE
    stride-1 pass with the four sub-pixel phases stacked on N (merge_transposed_weight) instead of four phase launches."""
    return os.environ.get("LWB_CONVT_MERGE", "1") != "0"


def merge_transposed_weight(wt):
    """IOHW [cin, cout, 3, 3] of ConvTranspose2d(k=3, s=2, p=1, output_padding=1) -> OIHW [4*cout, cin, 2, 2]: output
    channel block ph = 2a + b holds sub-pixel phase out[2y+a, 2x+b]; filter tap (dy, dx) reads in[y+dy, x+dx].
    Per axis: phase 0 uses k=1 at d=0; phase 1 uses k=2 at d=0 and k=0 at d=1 (oy = 2*iy - 1 + ky); the other 7 of the 16
    (phase, tap) blocks are zero."""
    cin, cout = wt.shape[0], wt.shape[1]
    k_of = ({0: 1}, {0: 2, 1: 0})
    out = torch.zeros((4 * cout, cin, 2, 2), dtype=torch.float32, device=wt.device)
    for a in range(2):
        for b in range(2):
            ph = 2 * a + b
            for dy, ky in k_of[a].items():
                for dx, kx in k_of[b].items():
                    out[ph * cout:(ph + 1) * cout, :, dy, dx] = wt[:, :, ky, kx].t().float()
    return out


def fold_head_weights(w_img, w_att):
    """[3,64,7,7] + [1,64,7,7] -> [32, 64, 7, 1]: output channel kx*4 + co of the (7 x 1) filter = column kx of head co
    (networks/generator.py:126-134; rows 28..31 are zero)."""
    w4 = torch.cat([w_img, w_att], dim=0).float()                      # [4, C, ky, kx]
    folded = w4.permute(3, 0, 1, 2).reshape(28, w4.shape[1], 7, 1)     # [kx*4+co, C, ky, 1]
    return torch.cat([folded, torch.zeros(4, w4.shape[1], 7, 1, dtype=folded.dtype, device=folded.device)], dim=0).contiguous()


def _align_corners():
    return K.default_align_corners()


def _halo_mode():
    """LWB_HALO: '0' (default) = CUDA-core 7x7 heads; 'auto' = halo plans for the row-K stem and the skippers + 7x7
    heads on tensor cores (N tile 16); 'all' = also the residual blocks.  Halo plans run through the same tap-group conv
    kernel as the others."""
    if precision_mode() == "fp16f8":
        return '0'                                         # halo plans have no fp8 path
    return os.environ.get("LWB_HALO", "0")


class NetworkBase(StreamOwner, nn.Module):
    """networks/networks.py:45-80."""

    def __init__(self):
        super(NetworkBase, self).__init__()
        self._name = 'BaseNetwork'

    @property
    def name(self):
        return self._name

    def init_weights(self):
        self.apply(self._weights_init_fn)
        self._lwb_invalidate()

    def _weights_init_fn(self, m):
        classname = m.__class__.__name__
        if classname.find('Conv') != -1:
            m.weight.data.normal_(0.0, 0.02)
            if hasattr(m.bias, 'data'):
                m.bias.data.fill_(0)
        elif classname.find('BatchNorm2d') != -1:
            m.weight.data.normal_(1.0, 0.02)
            m.bias.data.fill_(0)

    def _lwb_invalidate(self):
        _WEIGHTS_EPOCH[0] += 1                               # captured graphs keyed on it (imitator._chunk_step) are re-captured
        for m in self.modules():
            if hasattr(m, '_lwb_streams'):
                m._lwb_streams = {}

    def set_precision(self, mode):
        """Pin this network (and its sub-networks) to an operand mode regardless of LWB_PRECISION (None = follow the env)."""
        if mode not in (None, "fp16", "fp16x3", "fp16f8"):
            raise LwbError("precision must be fp16x3, fp16f8, fp16 or None")
        for m in self.modules():
            if isinstance(m, NetworkBase):
                m.__dict__['_lwb_precision'] = mode

    def range_flags(self):
        """-> list of int32[1] device tensors, one per stream used by the most recent pass: bit 0 = an activation left the e4m3 correction
        range (|x| >= 1024, fp16f8 precision degrades for those elements), bit 1 = the fp16 range (|x| >= 60000 / NaN),
        bit 2 = output-head pre-activations of +-8 and more in fp16f8 mode (its ~1e-4 relative end-to-end precision then
        no longer guarantees 1e-3 on the pixels: use fp16x3)."""
        live = []
        for m in self.modules():
            for st in getattr(m, '_lwb_streams', {}).values():
                live.append((getattr(st, 'pass_id', -1), st.range_flag))
        if not live:
            return []
        last = max(p for p, _ in live)                       # streams of other shapes / precisions keep the bits of older passes
        return [f for p, f in live if p == last]

    def range_flag_tensor(self):
        """One int32 device scalar = OR over the live streams' flags; None if no stream exists yet.  No host sync."""
        flags = self.range_flags()
        if not flags:
            return None
        if len(flags) == 1:
            return flags[0]
        acc = flags[0].clone()
        for f in flags[1:]:
            acc |= f
        return acc

    def range_status(self):
        """OR of range_flags() as a Python int (one device sync); streams reset their flag at the start of a pass."""
        flags = self.range_flags()
        if not flags:
            return 0
        bits = torch.stack([f.reshape(()) for f in flags]).cpu()
        out = 0
        for b in bits.tolist():
            out |= int(b)
        return out



class ResidualBlock(nn.Module):
    """networks/generator.py:8-20 (parameter holder)."""

    def __init__(self, dim_in, dim_out):
        super(ResidualBlock, self).__init__()
        self.main = nn.Sequential(
            nn.Conv2d(dim_in, dim_out, kernel_size=3, stride=1, padding=1, bias=False),
            nn.InstanceNorm2d(dim_out, affine=True),
            nn.ReLU(inplace=True),
            nn.Conv2d(dim_out, dim_out, kernel_size=3, stride=1, padding=1, bias=False),
            nn.InstanceNorm2d(dim_out, affine=True))

    def forward(self, x):
        raise LwbError("ResidualBlock runs only inside the fused generator streams")


# ------------------------------------------------------------------------------------------
# engine: one network bound to (batch, H, W, precision) -> persistent buffers + conv plans
# ------------------------------------------------------------------------------------------
class _Layer(object):
    """conv (+ InstanceNorm params) bound to buffers: plan + stats slot."""
    __slots__ = ("plan", "raw", "stats", "gamma", "beta", "w", "wsrc")


class _StreamBase(object):
    def __init__(self, B, H, W, dev, split):
        self.B, self.H, self.W, self.dev, self.split = B, H, W, dev, split
        self._stats_slots = []
        self._layers = []
        self._raw = {}
        self.ws = None

    def _raw_buf(self, h, w, c):
        key = (h, w, c)
        if key not in self._raw:
            self._raw[key] = torch.empty((self.B, h, w, c), dtype=torch.float32, device=self.dev)
        return self._raw[key]

    def _make_layer(self, conv, norm, x0, x1=None, stride=1, transposed=False, rowk=False, row_pitch=0, h=None, w=None,
                    halo=False, weight=None, pad=None, n_tile=0, pad_w=None):
        L = _Layer()
        wt = (weight if weight is not None else conv.weight).detach()
        L.wsrc = None
        if rowk:
            L.w = K.pack_conv_weight_rowk(wt, split=min(self.split, 1))       # the stem keeps the fp16 hi/lo input
            cout, kh, kw = wt.shape[0], wt.shape[2], wt.shape[3]
            d = K.make_conv_desc(self.B, h, w, 8, cout, kh, kw, stride=1, pad=kh // 2, split=min(self.split, 1),
                                 rowk=True, row_pitch=row_pitch, halo=halo)
        else:
            L.w = None
            cout = wt.shape[1] if transposed else wt.shape[0]
            kh, kw = wt.shape[2], wt.shape[3]
            merged = bool(transposed and _convt_merge() and cout <= 128 and cout % 32 == 0 and (kh, kw) == (3, 3))
            # packed in _finalize (one max|w| sync for the whole stream)
            L.wsrc = (merge_transposed_weight(wt), False) if merged else (wt, transposed)
            cin0 = x0[0].shape[3]
            cin1 = x1[0].shape[3] if x1 is not None else 0
            d = K.make_conv_desc(self.B, h, w, cin0, cout, kh, kw, stride=stride,
                                 pad=(pad if pad is not None else conv.padding[0]),
                                 cin1=cin1, transposed=transposed, split=self.split, halo=halo, n_tile=n_tile, pad_w=pad_w)
            if merged:
                d.transposed = 2                        # lwb_conv_desc: merged-phase weights
        L.raw = self._raw_buf(d.h_out, d.w_out, cout)
        L.stats = (len(self._stats_slots), cout)
        self._stats_slots.append(cout)
        L.gamma = norm.weight.detach().float().contiguous() if norm is not None else None
        L.beta = norm.bias.detach().float().contiguous() if norm is not None else None
        L.plan = (d, x0, x1)
        self._layers.append(L)
        return L

    def _finalize(self):
        cmax = max(max(self._stats_slots), 16)
        # InstanceNorm statistics of every layer + the operand-range flag share one buffer: one fill per pass
        nstat = len(self._stats_slots) * self.B * cmax * 2
        self._zero = torch.zeros(nstat * 8 + 4, dtype=torch.uint8, device=self.dev)
        self.stats = self._zero[:nstat * 8].view(torch.float64).view(len(self._stats_slots), self.B, cmax, 2)
        self.range_flag = self._zero[nstat * 8:].view(torch.int32)
        self.ws = torch.empty((self.B, cmax, 2), dtype=torch.float32, device=self.dev)
        pend = [L for L in self._layers if L.wsrc is not None]
        packed = pack_all([(L.wsrc[0], L.wsrc[1], None, None) for L in pend], self.split)
        for L, wp in zip(pend, packed):
            L.w, L.wsrc = wp, None
        for L in self._layers:
            slot, cout = L.stats
            # per-layer contiguous [B, cout, 2] view at the head of the slot (None: no norm follows)
            L.stats = None if self._stats_slots[slot] == 0 else \
                self.stats[slot].view(-1)[:self.B * cout * 2].view(self.B, cout, 2)
            d, x0, x1 = L.plan
            L.plan = K.ConvPlan(d, x0, x1, L.w, L.raw, L.stats)

    def _label_heads(self):
        """The folded heads issue N = 32 columns; their algorithmic work is the 7x7 x 64 -> 4 convolution."""
        L = getattr(self, 'head_layer', None)
        if L is not None and getattr(self, 'folded_kw', 7) == 7 and L.plan.desc.kw == 1:
            L.plan.flops = 2.0 * self.B * self.H * self.W * 49 * 64 * 4
            L.plan.label = "H7x7 64->4 @%d (7x1 filter, N = 7 cols x 4)" % self.H
            L.plan.prof_class = "heads"

    def begin_pass(self):
        """Zero the InstanceNorm statistics and the range flag (one fill)."""
        self._zero.zero_()
        self.pass_id = _PASS[0]

    def _conv_norm(self, L, out, relu, residual=None, warp_src=None, T=None, ac=False):
        L.plan.run()
        K.norm_act_nhwc(L.raw, L.stats, L.gamma, L.beta, relu, self.ws, residual=residual, warp_src=warp_src, T=T,
                        align_corners=ac, y_f32=out.f32, y_hi=out.hi, y_lo=out.lo, lo_format=1 if self.split == 2 else 0,
                        range_flag=self.range_flag)


class _UnetStream(_StreamBase):
    """ResUnetGenerator (networks/generator.py:68-184) bound to fixed shapes."""

    def __init__(self, net, B, H, W, dev, split, keep_f32=False):
        super(_UnetStream, self).__init__(B, H, W, dev, split)
        self.n_down, self.repeat = net.n_down, net.repeat_num
        nd = self.n_down
        if H % (1 << nd) or W % (1 << nd):
            raise LwbError("image size must be divisible by %d" % (1 << nd))
        self.keep_f32 = keep_f32
        # stem input: padded NHWC8 (3 px border top/left/bottom, 5 right) for the row-K 7x7 conv
        self.pitch = W + 8
        self.x_pad = Operands((B, H + 6, self.pitch, 8), dev, split)
        self.cin = net.encoders[0][0].weight.shape[1]
        if self.cin > 8:
            raise LwbError("stem supports at most 8 input channels")
        # encoders
        self.e, self.enc_layers = [], []
        c, h, w = net.encoders[0][0].weight.shape[0], H, W
        hm = _halo_mode()
        self.enc_layers.append(self._make_layer(net.encoders[0][0], net.encoders[0][1], self.x_pad.pair, rowk=True,
                                                row_pitch=self.pitch, h=H, w=W, halo=(hm != '0')))
        self.e.append(Operands((B, h, w, c), dev, split, f32=keep_f32))
        for i in range(1, nd + 1):
            self.enc_layers.append(self._make_layer(net.encoders[i][0], net.encoders[i][1], self.e[i - 1].pair,
                                                    stride=2, h=h, w=w))
            c, h, w = c * 2, h // 2, w // 2
            self.e.append(Operands((B, h, w, c), dev, split, f32=(keep_f32 or i == nd)))
        # resnets (ping-pong x buffers; h buffer for the mid activation)
        self.hb = Operands((B, h, w, c), dev, split)
        self.res_layers, self.res_out = [], []
        prev = self.e[nd]
        for i in range(self.repeat):
            out = Operands((B, h, w, c), dev, split, f32=True)
            l1 = self._make_layer(net.resnets[i].main[0], net.resnets[i].main[1], prev.pair, h=h, w=w, halo=(hm == 'all'))
            l2 = self._make_layer(net.resnets[i].main[3], net.resnets[i].main[4], self.hb.pair, h=h, w=w, halo=(hm == 'all'))
            self.res_layers.append((l1, l2))
            self.res_out.append(out)
            prev = out
        # decoders + skippers
        self.dec_layers, self.d_up, self.d_out = [], [], []
        for i in range(nd):
            up = Operands((B, h * 2, w * 2, c // 2), dev, split)
            ld = self._make_layer(net.decoders[i][0], net.decoders[i][1], prev.pair, stride=2, transposed=True, h=h, w=w)
            c, h, w = c // 2, h * 2, w * 2
            last = (i == nd - 1)
            tc_heads = (hm != '0') or (_tc_heads() and c == 64)
            out = Operands((B, h, w, c), dev, split, f32=(last and not tc_heads), half=(not last or tc_heads))
            ls = self._make_layer(net.skippers[i][0], net.skippers[i][1], self.e[nd - 1 - i].pair, x1=up.pair, h=h, w=w,
                                  halo=(hm != '0'))
            self.dec_layers.append((ld, ls))
            self.d_up.append(up)
            self.d_out.append(out)
            prev = out
        w_img, w_att = net.img_reg[0].weight.detach(), net.attetion_reg[0].weight.detach()
        self.head_layer = None
        self.folded_kw = 0
        if hm == '0' and _tc_heads() and c == 64:
            # img_reg (64->3) + attetion_reg (64->1): a 7 x 1 filter with N = 7 columns x 4 channels (-> 32) on the tensor
            # cores; the composite kernel adds the seven column partials of every pixel (lwb_heads_composite, folded_kw)
            self.head_layer = self._make_layer(None, None, prev.pair, h=H, w=W, weight=fold_head_weights(w_img, w_att),
                                               pad=3, pad_w=0, n_tile=32)
            self._stats_slots[-1] = 0
            self.head_raw = self.head_layer.raw
            self.folded_kw = 7
        elif hm != '0':
            # img_reg (64->3) + attetion_reg (64->1) as one 7x7 conv padded to 16 output channels on the
            # tensor cores (halo variant, N tile 16); channels 0..3 are consumed by the composite kernel
            w16 = torch.cat([w_img, w_att, torch.zeros(12, *w_img.shape[1:], device=w_img.device, dtype=w_img.dtype)], dim=0)
            self.head_layer = self._make_layer(None, None, prev.pair, h=H, w=W, halo=True, weight=w16, pad=3, n_tile=16)
            self._stats_slots[-1] = 0          # no InstanceNorm after the heads: no statistics
            self.head_raw = self.head_layer.raw
        else:
            self.w4 = K.pack_head_weights(w_img, w_att)
            self.head_raw = torch.empty((B, H, W, 4), dtype=torch.float32, device=dev)
        self._finalize()
        self._label_heads()

    # ---- pieces -------------------------------------------------------------------------
    def load_input(self, x):
        if tuple(x.shape) != (self.B, self.cin, self.H, self.W) or x.dtype != torch.float32:
            raise LwbError("unexpected input %s (stream built for %s)" % (tuple(x.shape), (self.B, self.cin, self.H, self.W)))
        K.nchw_to_nhwc_split(x.contiguous(), c_pad=8, pad_hw=(3, 3, 3, 5), hi=self.x_pad.hi, lo=self.x_pad.lo)

    def encode(self, warp_srcs=None, T=None, ac=False, upto=None):
        """encoders 0..n_down; warp_srcs[i] (NHWC fp32, i >= 1) is LWB-added after encoder i."""
        self.begin_pass()
        self._conv_norm(self.enc_layers[0], self.e[0], True)
        for i in range(1, self.n_down + 1):
            src = warp_srcs[i] if warp_srcs is not None else None
            if isinstance(src, (list, tuple)):          # swap(): two warps per site
                self._conv_norm(self.enc_layers[i], self.e[i], True, warp_src=src[0][0], T=src[0][1], ac=ac)
                self._add_warp(self.e[i], src[1][0], src[1][1], ac)
            else:
                self._conv_norm(self.enc_layers[i], self.e[i], True, warp_src=src, T=T, ac=ac)

    def _add_warp(self, act, src, T, ac):
        if act.f32 is None:
            raise LwbError("second warp needs an fp32 activation")
        K.norm_act_nhwc(act.f32, None, None, None, False, self.ws, warp_src=src, T=T, align_corners=ac,
                        y_f32=act.f32, y_hi=act.hi, y_lo=act.lo, lo_format=1 if self.split == 2 else 0,
                        range_flag=self.range_flag)

    def resnets(self, warp_srcs=None, T=None, ac=False):
        x = self.e[self.n_down]
        for i, (l1, l2) in enumerate(self.res_layers):
            self._conv_norm(l1, self.hb, True)
            src = warp_srcs[i] if warp_srcs is not None else None
            if isinstance(src, (list, tuple)):
                self._conv_norm(l2, self.res_out[i], False, residual=x.f32, warp_src=src[0][0], T=src[0][1], ac=ac)
                self._add_warp(self.res_out[i], src[1][0], src[1][1], ac)
            else:
                self._conv_norm(l2, self.res_out[i], False, residual=x.f32, warp_src=src, T=T, ac=ac)
            x = self.res_out[i]

    def decode(self):
        for i, (ld, ls) in enumerate(self.dec_layers):
            self._conv_norm(ld, self.d_up[i], True)
            self._conv_norm(ls, self.d_out[i], True)

    def heads(self, bg=None, want_color=True, want_mask=True, **out):
        if self.head_layer is not None:
            self.head_layer.plan.run()
        else:
            K.conv7x7_heads_nhwc(self.d_out[-1].f32, self.w4, out=self.head_raw)
        return K.heads_composite(self.head_raw, bg, want_color=want_color, want_mask=want_mask, folded_kw=self.folded_kw,
                                 range_flag=self.range_flag if self.split == 2 else None, **out)

    def encoder_outs_nchw(self):
        outs = []
        for a in self.e:
            t = K.nhwc_to_nchw(a.f32)
            t._lwb_nhwc = a.f32.clone()
            outs.append(t)
        return outs

    def resnet_outs_nchw(self):
        outs = []
        for a in self.res_out:
            t = K.nhwc_to_nchw(a.f32)
            t._lwb_nhwc = a.f32.clone()
            outs.append(t)
        return outs


class _ResnetStream(_StreamBase):
    """ResNetGenerator (networks/generator.py:23-65, the BG net) bound to fixed shapes."""

    def __init__(self, net, B, H, W, dev, split):
        super(_ResnetStream, self).__init__(B, H, W, dev, split)
        layers = list(net.model)
        nd, rep = net._n_down, net._repeat_num
        self.pitch = W + 8
        self.x_pad = Operands((B, H + 6, self.pitch, 8), dev, split)
        self.cin = layers[0].weight.shape[1]
        if self.cin > 8:
            raise LwbError("stem supports at most 8 input channels")
        self.seq = []
        i = 0
        c, h, w = layers[0].weight.shape[0], H, W
        out = Operands((B, h, w, c), dev, split)
        self.seq.append(("cn", self._make_layer(layers[0], layers[1], self.x_pad.pair, rowk=True, row_pitch=self.pitch, h=H, w=W), out, True, None))
        prev = out
        i += 3
        for k in range(nd):
            out = Operands((B, h // 2, w // 2, c * 2), dev, split, f32=(k == nd - 1))
            self.seq.append(("cn", self._make_layer(layers[i], layers[i + 1], prev.pair, stride=2, h=h, w=w), out, True, None))
            c, h, w = c * 2, h // 2, w // 2
            prev = out
            i += 3
        hb = Operands((B, h, w, c), dev, split)
        for k in range(rep):
            blk = layers[i]
            out = Operands((B, h, w, c), dev, split, f32=True)
            self.seq.append(("cn", self._make_layer(blk.main[0], blk.main[1], prev.pair, h=h, w=w), hb, True, None))
            self.seq.append(("cn", self._make_layer(blk.main[3], blk.main[4], hb.pair, h=h, w=w), out, False, prev))
            prev = out
            i += 1
        for k in range(nd):
            last = (k == nd - 1)
            tc_heads = _tc_heads() and c // 2 == 64
            out = Operands((B, h * 2, w * 2, c // 2), dev, split, f32=(last and not tc_heads), half=(not last or tc_heads))
            self.seq.append(("cn", self._make_layer(layers[i], layers[i + 1], prev.pair, stride=2, transposed=True, h=h, w=w), out, True, None))
            c, h, w = c // 2, h * 2, w * 2
            prev = out
            i += 3
        self.final = prev
        w_img = layers[i].weight.detach()
        self.head_layer = None
        if _tc_heads() and c == 64:
            self.head_layer = self._make_layer(None, None, prev.pair, h=H, w=W, pad=3, pad_w=0, n_tile=32,
                                               weight=fold_head_weights(w_img, torch.zeros_like(w_img[:1])))
            self._stats_slots[-1] = 0
            self.head_raw = self.head_layer.raw
        else:
            self.w4 = K.pack_head_weights(w_img, torch.zeros_like(w_img[:1]))
            self.head_raw = torch.empty((B, H, W, 4), dtype=torch.float32, device=dev)
        self._finalize()
        self._label_heads()

    def run(self, x):
        if tuple(x.shape) != (self.B, self.cin, self.H, self.W):
            raise LwbError("unexpected input shape %s" % (tuple(x.shape),))
        K.nchw_to_nhwc_split(x.float().contiguous(), c_pad=8, pad_hw=(3, 3, 3, 5), hi=self.x_pad.hi, lo=self.x_pad.lo)
        self.begin_pass()
        for _, L, out, relu, res in self.seq:
            self._conv_norm(L, out, relu, residual=(res.f32 if res is not None else None))
        if self.head_layer is not None:
            self.head_layer.plan.run()
        else:
            K.conv7x7_heads_nhwc(self.final.f32, self.w4, out=self.head_raw)
        color, _, _ = K.heads_composite(self.head_raw, None, want_color=True, want_mask=False,
                                        folded_kw=7 if self.head_layer is not None else 0)
        return color


def profile_streams(warm_fn, run_fn):
    """Instrumented passes: CUDA events around every kernel class (bench.py roofline / breakdown).
    -> {"passes": n, "conv": {"ms", "flops", "n"}, "norm": {"ms", "bytes", "n"}, "heads"/"correspond"/"input": {"ms", ...}}"""
    warm_fn()
    torch.cuda.synchronize()
    K.profile_begin()
    n = len(run_fn())
    raw = K.profile_end()
    out = {"passes": n}
    for cls in ("conv", "norm", "heads", "correspond", "input"):
        r = raw.get(cls, {"ms": 0.0, "work": 0.0, "n": 0})
        out[cls] = {"ms": r["ms"], "n": r["n"], ("flops" if cls in ("conv", "heads") else "bytes"): r["work"]}
    out["layers"] = {k: {"ms": v["ms"] / n, "n": v["n"] / n, "work": v["work"] / n} for k, v in raw.items() if "/" in k}
    return out


def _stream_for(mod, cls, key, *args, **kw):
    """The generator networks' per-shape stream cache: the 8 most recently used shapes (each holds ~GBs at B=16)."""
    return stream_for(mod, cls, key, *args, limit=8, **kw)


def _nhwc_of(t):
    """NHWC fp32 twin of an NCHW feature (cached on the tensor by encode_src / inference)."""
    cached = getattr(t, '_lwb_nhwc', None)
    if cached is not None:
        return cached
    return t.permute(0, 2, 3, 1).contiguous()


class ResNetGenerator(NetworkBase):
    """Generator. Encoder-Decoder Architecture (networks/generator.py:23-65)."""

    def __init__(self, conv_dim=64, c_dim=5, repeat_num=9, k_size=4, n_down=2):
        super(ResNetGenerator, self).__init__()
        self._name = 'resnet_generator'
        self._n_down, self._repeat_num = n_down, repeat_num
        if k_size != 3:
            raise LwbError("the conv engine implements k_size=3 (what ImpersonatorGenerator uses)")
        layers = []
        layers.append(nn.Conv2d(c_dim, conv_dim, kernel_size=7, stride=1, padding=3, bias=False))
        layers.append(nn.InstanceNorm2d(conv_dim, affine=True))
        layers.append(nn.ReLU(inplace=True))
        curr_dim = conv_dim
        for i in range(n_down):
            layers.append(nn.Conv2d(curr_dim, curr_dim * 2, kernel_size=k_size, stride=2, padding=1, bias=False))
            layers.append(nn.InstanceNorm2d(curr_dim * 2, affine=True))
            layers.append(nn.ReLU(inplace=True))
            curr_dim = curr_dim * 2
        for i in range(repeat_num):
            layers.append(ResidualBlock(dim_in=curr_dim, dim_out=curr_dim))
        for i in range(n_down):
            layers.append(nn.ConvTranspose2d(curr_dim, curr_dim // 2, kernel_size=k_size, stride=2, padding=1,
                                             output_padding=1, bias=False))
            layers.append(nn.InstanceNorm2d(curr_dim // 2, affine=True))
            layers.append(nn.ReLU(inplace=True))
            curr_dim = curr_dim // 2
        layers.append(nn.Conv2d(curr_dim, 3, kernel_size=7, stride=1, padding=3, bias=False))
        layers.append(nn.Tanh())
        self.model = nn.Sequential(*layers)

    @torch.no_grad()
    def forward(self, x, c=None):
        if c is not None:
            c = c.unsqueeze(2).unsqueeze(3)
            c = c.expand(c.size(0), c.size(1), x.size(2), x.size(3))
            x = torch.cat([x, c], dim=1)
        B, _, H, W = x.shape
        split = split_mode(self)
        st = _stream_for(self, _ResnetStream, ('bg', B, H, W, split), B, H, W, x.device, split)
        return st.run(x)


class ResUnetGenerator(NetworkBase):
    """Generator. Encoder-Decoder Architecture (networks/generator.py:68-184)."""

    def __init__(self, conv_dim=64, c_dim=5, repeat_num=6, k_size=4, n_down=2):
        super(ResUnetGenerator, self).__init__()
        self._name = 'resunet_generator'
        self.repeat_num = repeat_num
        self.n_down = n_down
        if k_size != 3:
            raise LwbError("the conv engine implements k_size=3 (what ImpersonatorGenerator uses)")
        encoders = []
        encoders.append(nn.Sequential(
            nn.Conv2d(c_dim, conv_dim, kernel_size=7, stride=1, padding=3, bias=False),
            nn.InstanceNorm2d(conv_dim, affine=True),
            nn.ReLU(inplace=True)))
        curr_dim = conv_dim
        for i in range(n_down):
            encoders.append(nn.Sequential(
                nn.Conv2d(curr_dim, curr_dim * 2, kernel_size=k_size, stride=2, padding=1, bias=False),
                nn.InstanceNorm2d(curr_dim * 2, affine=True),
                nn.ReLU(inplace=True)))
            curr_dim = curr_dim * 2
        self.encoders = nn.Sequential(*encoders)
        resnets = []
        for i in range(repeat_num):
            resnets.append(ResidualBlock(dim_in=curr_dim, dim_out=curr_dim))
        self.resnets = nn.Sequential(*resnets)
        decoders, skippers = [], []
        for i in range(n_down):
            decoders.append(nn.Sequential(
                nn.ConvTranspose2d(curr_dim, curr_dim // 2, kernel_size=k_size, stride=2, padding=1, output_padding=1, bias=False),
                nn.InstanceNorm2d(curr_dim // 2, affine=True),
                nn.ReLU(inplace=True)))
            skippers.append(nn.Sequential(
                nn.Conv2d(curr_dim, curr_dim // 2, kernel_size=k_size, stride=1, padding=1, bias=False),
                nn.InstanceNorm2d(curr_dim // 2, affine=True),
                nn.ReLU(inplace=True)))
            curr_dim = curr_dim // 2
        self.decoders = nn.Sequential(*decoders)
        self.skippers = nn.Sequential(*skippers)
        layers = []
        layers.append(nn.Conv2d(curr_dim, 3, kernel_size=7, stride=1, padding=3, bias=False))
        layers.append(nn.Tanh())
        self.img_reg = nn.Sequential(*layers)
        layers = []
        layers.append(nn.Conv2d(curr_dim, 1, kernel_size=7, stride=1, padding=3, bias=False))
        layers.append(nn.Sigmoid())
        self.attetion_reg = nn.Sequential(*layers)

    def _stream(self, x, keep_f32, tag):
        B, _, H, W = x.shape
        split = split_mode(self)
        return _stream_for(self, _UnetStream, (tag, B, H, W, split, keep_f32), B, H, W, x.device, split, keep_f32=keep_f32)

    @torch.no_grad()
    def inference(self, x):
        """encoder_outs [4], resnet_outs [6] as NCHW fp32 (networks/generator.py:136-147)."""
        st = self._stream(x, True, 'inference')
        st.load_input(x.float())
        st.encode()
        st.resnets()
        return st.encoder_outs_nchw(), st.resnet_outs_nchw()

    @torch.no_grad()
    def forward(self, x):
        st = self._stream(x, False, 'forward')
        st.load_input(x.float())
        st.encode()
        st.resnets()
        st.decode()
        color, mask, _ = st.heads()
        return color, mask

    def encode(self, x):
        return self.inference(x)[0]

    def decode(self, x, encoder_outs):
        raise LwbError("decode() on detached tensors is not part of the inference hot path; use forward()/inference()")

    def regress(self, x):
        raise LwbError("regress() on detached tensors is not part of the inference hot path; use forward()")


class ImpersonatorGenerator(NetworkBase):
    """Generator. Encoder-Decoder Architecture (networks/generator.py:187-320)."""

    def __init__(self, bg_dim, src_dim, tsf_dim, conv_dim=64, repeat_num=6):
        super(ImpersonatorGenerator, self).__init__()
        self._name = 'impersonator_generator'
        self.n_down = 3
        self.repeat_num = repeat_num
        self.bg_model = ResNetGenerator(conv_dim=conv_dim, c_dim=bg_dim, repeat_num=repeat_num, k_size=3, n_down=self.n_down)
        self.src_model = ResUnetGenerator(conv_dim=conv_dim, c_dim=src_dim, repeat_num=repeat_num, k_size=3, n_down=self.n_down)
        self.tsf_model = ResUnetGenerator(conv_dim=conv_dim, c_dim=tsf_dim, repeat_num=repeat_num, k_size=3, n_down=self.n_down)

    @torch.no_grad()
    def forward(self, bg_inputs, src_inputs, tsf_inputs, T):
        img_bg = self.bg_model(bg_inputs)
        src_img, src_mask, tsf_img, tsf_mask = self.infer_front(src_inputs, tsf_inputs, T)
        return img_bg, src_img, src_mask, tsf_img, tsf_mask

    def encode_src(self, src_inputs):
        _new_pass()
        return self.src_model.inference(src_inputs)

    @torch.no_grad()
    def infer_front(self, src_inputs, tsf_inputs, T):
        ac = _align_corners()
        _new_pass()
        T = T.float().contiguous()
        src = self.src_model._stream(src_inputs, True, 'front')
        src.load_input(src_inputs.float())
        src.encode()
        src.resnets()
        tsf = self.tsf_model._stream(tsf_inputs, False, 'front')
        tsf.load_input(tsf_inputs.float())
        tsf.encode(warp_srcs=[None] + [a.f32 for a in src.e[1:]], T=T, ac=ac)
        tsf.resnets(warp_srcs=[a.f32 for a in src.res_out], T=T, ac=ac)
        src.decode()
        src_img, src_mask, _ = src.heads()
        tsf.decode()
        tsf_img, tsf_mask, _ = tsf.heads()
        return src_img, src_mask, tsf_img, tsf_mask

    @torch.no_grad()
    def swap(self, tsf_inputs, src_encoder_outs12, src_encoder_outs21, src_resnet_outs12, src_resnet_outs21, T12, T21, bg=None):
        """networks/generator.py:245-275.  With ``bg`` (extension) also returns the composite m*bg + (1-m)*color of
        models/swapper.py:268-269 from the head kernel."""
        ac = _align_corners()
        _new_pass()
        T12, T21 = T12.float().contiguous(), T21.float().contiguous()
        tsf = self.tsf_model._stream(tsf_inputs, True, 'swap')
        tsf.load_input(tsf_inputs.float())
        enc = [None] + [((_nhwc_of(a), T12), (_nhwc_of(b), T21)) for a, b in zip(src_encoder_outs12[1:], src_encoder_outs21[1:])]
        res = [((_nhwc_of(a), T12), (_nhwc_of(b), T21)) for a, b in zip(src_resnet_outs12, src_resnet_outs21)]
        tsf.encode(warp_srcs=enc, ac=ac)
        tsf.resnets(warp_srcs=res, ac=ac)
        tsf.decode()
        tsf_img, tsf_mask, pred = tsf.heads(bg)
        if bg is not None:
            return tsf_img, tsf_mask, pred
        return tsf_img, tsf_mask

    @torch.no_grad()
    def inference(self, src_encoder_outs, src_resnet_outs, tsf_inputs, T, bg=None, pred_hwc=None, pred_u8=None):
        """networks/generator.py:277-301.  With ``bg`` also returns the composite of
        models/imitator.py:331 as a third value (fused into the head kernel); ``pred_hwc`` / ``pred_u8``
        (caller-allocated [B,H,W,3] float32 / uint8-BGR) receive the same frames in the layouts of the output
        path (models/imitator.py:178-180, utils/cv_utils.py:23-36) from that launch."""
        ac = _align_corners()
        _new_pass()
        if (pred_hwc is not None or pred_u8 is not None) and bg is None:
            raise LwbError("pred_hwc / pred_u8 need bg (they hold the composite)")
        tsf_inputs = tsf_inputs.float().contiguous()
        T = T.float().contiguous()
        enc_w = [None] + [_nhwc_of(a) for a in src_encoder_outs[1:]]
        res_w = [_nhwc_of(a) for a in src_resnet_outs]
        B = tsf_inputs.shape[0]
        nsub = _sub_batches(B, enc_w, res_w, bg)

        def run(tag, x, Tx, outs):
            tsf = self.tsf_model._stream(x, False, tag)
            tsf.load_input(x)
            tsf.encode(warp_srcs=enc_w, T=Tx, ac=ac)
            tsf.resnets(warp_srcs=res_w, T=Tx, ac=ac)
            tsf.decode()
            return tsf.heads(bg, **outs)

        if nsub == 1:
            outs = {}
            if pred_hwc is not None or pred_u8 is not None:
                outs = dict(pred_hwc=pred_hwc, pred_u8=pred_u8)
            color, mask, pred = run('inference', tsf_inputs, T, outs)
        else:
            # LWB_STREAMS sub-batches on side streams: the HBM-bound kernels of one sub-batch (InstanceNorm / warp, heads
            # composite, input packing) co-run with the tensor-bound convolutions of the other, and the second wave of
            # the twelve 512-channel layers (128 tile pairs on 74 SM pairs) is filled by the other sub-batch's tiles.
            _, _, H, W = tsf_inputs.shape
            dev = tsf_inputs.device
            color = torch.empty((B, 3, H, W), dtype=torch.float32, device=dev)
            mask = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
            pred = torch.empty((B, 3, H, W), dtype=torch.float32, device=dev) if bg is not None else None
            side = self.__dict__.setdefault('_lwb_side_streams', {})
            cur = torch.cuda.current_stream(dev)
            ready = torch.cuda.Event()
            ready.record(cur)
            step = B // nsub
            for i in range(nsub):
                if (dev, i) not in side:
                    side[(dev, i)] = torch.cuda.Stream(device=dev)
                st = side[(dev, i)]
                st.wait_event(ready)
                a, b = i * step, (i + 1) * step
                with torch.cuda.stream(st):
                    outs = dict(color=color[a:b], mask=mask[a:b])
                    if pred is not None:
                        outs['pred'] = pred[a:b]
                    if pred_hwc is not None:
                        outs['pred_hwc'] = pred_hwc[a:b]
                    if pred_u8 is not None:
                        outs['pred_u8'] = pred_u8[a:b]
                    run('inference#%d' % i, tsf_inputs[a:b], T[a:b], outs)
                    done = torch.cuda.Event()
                    done.record(st)
                cur.wait_event(done)
        if bg is not None:
            return color, mask, pred
        return color, mask

    def resize_trans(self, x, T):
        raise LwbError("resize_trans is fused into the warp kernels; call transform()/stn()")

    @torch.no_grad()
    def stn(self, x, T):
        return K.warp_nchw(x.float().contiguous(), T.float().contiguous(), align_corners=_align_corners())

    @torch.no_grad()
    def transform(self, x, T):
        return K.warp_nchw(x.float().contiguous(), T.float().contiguous(), align_corners=_align_corners())
