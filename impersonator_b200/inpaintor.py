"""Host-side mirror of networks/inpaintor.py (DeepFill-v2 style ``InpaintSANet``), the default
background network of ``Imitator.personalize`` (models/imitator.py:48-52,124-125; once per source).

Same module tree and ``state_dict`` keys as the reference (322 tensors incl. BatchNorm running
stats): ``GatedConv2dWithActivation`` (conv2d, mask_conv2d, batch_norm2d), ``GatedDeConv2dWithActivation``
(nearest 2x + gated conv), ``SelfAttention`` (query/key/value 1x1 convs, gamma), ``InpaintSANet``
(coarse_net 17 / refine_conv_net 11 / refine_attn / refine_upsample_net 7).

Execution (``InpaintSANet.forward``): the whole network is bound once per input shape to persistent NHWC
buffers (``_InpaintStream``).  Every gated layer = ONE wgmma conv-engine plan over the stacked
[conv2d ; mask_conv2d] filters (bias, dilation 2-16, 5x5, 4x4 stride 2; channels zero-padded to the engine's
64-wide K chunks / 16-wide N) + the fused gate / BatchNorm / nearest-2x / clamp epilogue
(lwb_gated_act_nhwc) that emits the next layer's operands directly; the 4096 x 4096 self-attention is the
stacked 1x1 q/k/v convolution on the engine + a flash-style fp32 kernel (lwb_self_attention_nhwc).  No
library GEMM / softmax is left on this path.  It runs once per source image, off the per-frame loop.
The sub-modules stay callable on their own (``GatedConv2dWithActivation.forward`` etc.: the fp32 direct
convolution + lwb_gated_bn_nchw), which is what unit tests of single layers use.
"""
import numpy as np
import torch
import torch.nn as nn

from . import kernels as K
from ._lib import LwbError
from .binding import Operands, PlanBinder, StreamOwner, bn_affine, lo_format, split_mode, stream_for


def get_pad(in_, ksize, stride, atrous=1):
    """networks/inpaintor.py:7-9."""
    out_ = np.ceil(float(in_) / stride)
    return int(((out_ - 1) * stride + atrous * (ksize - 1) + 1 - in_) / 2)


class GatedConv2dWithActivation(nn.Module):
    """phi(f(I)) * sigmoid(g(I)), then BatchNorm (networks/inpaintor.py:12-47)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True,
                 batch_norm=True, activation=torch.nn.LeakyReLU(0.2, inplace=True)):
        super(GatedConv2dWithActivation, self).__init__()
        if groups != 1:
            raise LwbError("grouped gated convs are not used by InpaintSANet")
        self.batch_norm = batch_norm
        self.activation = activation
        self.conv2d = torch.nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)
        self.mask_conv2d = torch.nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)
        self.batch_norm2d = torch.nn.BatchNorm2d(out_channels)
        self.sigmoid = torch.nn.Sigmoid()
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight)
        self._packed = None

    def _pack(self):
        dev = self.conv2d.weight.device
        if self._packed is None or self._packed[0].device != dev:
            w = torch.cat([self.conv2d.weight, self.mask_conv2d.weight], dim=0).detach().float().contiguous()
            b = None
            if self.conv2d.bias is not None:
                b = torch.cat([self.conv2d.bias, self.mask_conv2d.bias]).detach().float().contiguous()
            scale = shift = None
            if self.batch_norm:
                bn = self.batch_norm2d
                scale = (bn.weight / torch.sqrt(bn.running_var + bn.eps)).detach().float().contiguous()
                shift = (bn.bias - bn.running_mean * scale).detach().float().contiguous()
            self._packed = (w, b, scale, shift)
        return self._packed

    @torch.no_grad()
    def forward(self, input):
        if self.training:
            raise LwbError("the lwb_b200 path is inference-only (eval-mode BatchNorm)")
        w, b, scale, shift = self._pack()
        ab = K.conv2d_direct_nchw(input.float().contiguous(), w, b, stride=self.conv2d.stride[0],
                                  pad=self.conv2d.padding[0], dil=self.conv2d.dilation[0])
        act = 0 if self.activation is None else 2
        return K.gated_bn_nchw(ab, act, scale, shift)


class GatedDeConv2dWithActivation(nn.Module):
    """nearest 2x resize + gated conv (networks/inpaintor.py:50-68)."""

    def __init__(self, scale_factor, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, batch_norm=True, activation=torch.nn.LeakyReLU(0.2, inplace=True)):
        super(GatedDeConv2dWithActivation, self).__init__()
        self.conv2d = GatedConv2dWithActivation(in_channels, out_channels, kernel_size, stride, padding, dilation, groups,
                                                bias, batch_norm, activation)
        self.scale_factor = scale_factor

    @torch.no_grad()
    def forward(self, input):
        n, c, h, w = input.shape
        x = input[:, :, :, None, :, None].expand(n, c, h, 2, w, 2).reshape(n, c, 2 * h, 2 * w)   # nearest x2 (:67)
        return self.conv2d(x)


class SelfAttention(nn.Module):
    """networks/inpaintor.py:71-107."""

    def __init__(self, in_dim, activation, with_attn=False):
        super(SelfAttention, self).__init__()
        self.chanel_in = in_dim
        self.activation = activation
        self.with_attn = with_attn
        self.query_conv = nn.Conv2d(in_channels=in_dim, out_channels=in_dim // 8, kernel_size=1)
        self.key_conv = nn.Conv2d(in_channels=in_dim, out_channels=in_dim // 8, kernel_size=1)
        self.value_conv = nn.Conv2d(in_channels=in_dim, out_channels=in_dim, kernel_size=1)
        self.gamma = nn.Parameter(torch.zeros(1))
        self.softmax = nn.Softmax(dim=-1)

    @torch.no_grad()
    def forward(self, x):
        b, C, width, height = x.size()
        x = x.float().contiguous()
        conv = lambda m: K.conv2d_direct_nchw(x, m.weight.detach().float().contiguous(), m.bias.detach().float().contiguous())
        q = conv(self.query_conv).view(b, -1, width * height).permute(0, 2, 1)
        k = conv(self.key_conv).view(b, -1, width * height)
        attention = torch.softmax(torch.bmm(q, k), dim=-1)                   # library GEMM + softmax (cold path)
        v = conv(self.value_conv).view(b, -1, width * height)
        out = torch.bmm(v, attention.permute(0, 2, 1)).view(b, C, width, height)
        out = self.gamma * out + x
        return (out, attention) if self.with_attn else out


class InpaintSANet(StreamOwner, torch.nn.Module):
    """networks/inpaintor.py:110-202."""

    def __init__(self, c_dim=5):
        super(InpaintSANet, self).__init__()
        cnum = 32
        G, D = GatedConv2dWithActivation, GatedDeConv2dWithActivation
        self.coarse_net = nn.Sequential(
            G(c_dim, cnum, 5, 1, padding=get_pad(256, 5, 1)),
            G(cnum, 2 * cnum, 4, 2, padding=get_pad(256, 4, 2)),
            G(2 * cnum, 2 * cnum, 3, 1, padding=get_pad(128, 3, 1)),
            G(2 * cnum, 4 * cnum, 4, 2, padding=get_pad(128, 4, 2)),
            G(4 * cnum, 4 * cnum, 3, 1, padding=get_pad(64, 3, 1)),
            G(4 * cnum, 4 * cnum, 3, 1, padding=get_pad(64, 3, 1)),
            G(4 * cnum, 4 * cnum, 3, 1, dilation=2, padding=get_pad(64, 3, 1, 2)),
            G(4 * cnum, 4 * cnum, 3, 1, dilation=4, padding=get_pad(64, 3, 1, 4)),
            G(4 * cnum, 4 * cnum, 3, 1, dilation=8, padding=get_pad(64, 3, 1, 8)),
            G(4 * cnum, 4 * cnum, 3, 1, dilation=16, padding=get_pad(64, 3, 1, 16)),
            G(4 * cnum, 4 * cnum, 3, 1, padding=get_pad(64, 3, 1)),
            G(4 * cnum, 4 * cnum, 3, 1, padding=get_pad(64, 3, 1)),
            D(2, 4 * cnum, 2 * cnum, 3, 1, padding=get_pad(128, 3, 1)),
            G(2 * cnum, 2 * cnum, 3, 1, padding=get_pad(128, 3, 1)),
            D(2, 2 * cnum, cnum, 3, 1, padding=get_pad(256, 3, 1)),
            G(cnum, cnum // 2, 3, 1, padding=get_pad(256, 3, 1)),
            G(cnum // 2, 3, 3, 1, padding=get_pad(128, 3, 1), activation=None))
        self.refine_conv_net = nn.Sequential(
            G(c_dim, cnum, 5, 1, padding=get_pad(256, 5, 1)),
            G(cnum, cnum, 4, 2, padding=get_pad(256, 4, 2)),
            G(cnum, 2 * cnum, 3, 1, padding=get_pad(128, 3, 1)),
            G(2 * cnum, 2 * cnum, 4, 2, padding=get_pad(128, 4, 2)),
            G(2 * cnum, 4 * cnum, 3, 1, padding=get_pad(64, 3, 1)),
            G(4 * cnum, 4 * cnum, 3, 1, padding=get_pad(64, 3, 1)),
            G(4 * cnum, 4 * cnum, 3, 1, padding=get_pad(64, 3, 1)),
            G(4 * cnum, 4 * cnum, 3, 1, dilation=2, padding=get_pad(64, 3, 1, 2)),
            G(4 * cnum, 4 * cnum, 3, 1, dilation=4, padding=get_pad(64, 3, 1, 4)),
            G(4 * cnum, 4 * cnum, 3, 1, dilation=8, padding=get_pad(64, 3, 1, 8)),
            G(4 * cnum, 4 * cnum, 3, 1, dilation=16, padding=get_pad(64, 3, 1, 16)))
        self.refine_attn = SelfAttention(4 * cnum, 'relu', with_attn=False)
        self.refine_upsample_net = nn.Sequential(
            G(4 * cnum, 4 * cnum, 3, 1, padding=get_pad(64, 3, 1)),
            G(4 * cnum, 4 * cnum, 3, 1, padding=get_pad(64, 3, 1)),
            D(2, 4 * cnum, 2 * cnum, 3, 1, padding=get_pad(128, 3, 1)),
            G(2 * cnum, 2 * cnum, 3, 1, padding=get_pad(128, 3, 1)),
            D(2, 2 * cnum, cnum, 3, 1, padding=get_pad(256, 3, 1)),
            G(cnum, cnum // 2, 3, 1, padding=get_pad(256, 3, 1)),
            G(cnum // 2, 3, 3, 1, padding=get_pad(256, 3, 1), activation=None))

    def _stream(self, x):
        B, _, H, W = x.shape
        split = split_mode(self)
        return stream_for(self, _InpaintStream, (B, H, W, split), B, H, W, x.device, split, limit=2)

    @torch.no_grad()
    def forward(self, imgs, masks, only_out=False, only_x=False):
        if self.training:
            raise LwbError("the lwb_b200 path is inference-only (eval-mode BatchNorm)")
        if not imgs.is_cuda:
            raise LwbError("InpaintSANet runs on CUDA tensors only (no CPU fallback)")
        imgs, masks = imgs.float(), masks.float()
        st = self._stream(imgs)
        masked_imgs = imgs * (1 - masks) + masks
        coarse_x = st.run_coarse(torch.cat([masked_imgs, masks], dim=1))          # clamp fused into the last epilogue (:187)
        masked_imgs = imgs * (1 - masks) + coarse_x * masks
        x = st.run_refine(torch.cat([masked_imgs, masks], dim=1))                 # conv net + attention + upsample net, clamped (:196)
        comp_imgs = x * masks + imgs * (1 - masks)
        if only_out:
            return comp_imgs
        if only_x:
            return x
        return coarse_x, x, comp_imgs


def _ceil_to(v, m):
    return (v + m - 1) // m * m


class _InpaintStream(object):
    """InpaintSANet bound to (batch, H, W, precision): NHWC operand buffers, conv plans over the stacked gated filters,
    folded BatchNorms.  Channel counts (4, 16, 32) below the engine's 64-wide K chunk are zero-padded."""

    def __init__(self, net, B, H, W, dev, split):
        if H % 4 or W % 4:
            raise LwbError("InpaintSANet needs H, W divisible by 4")
        self.B, self.H, self.W, self.dev, self.split = B, H, W, dev, split
        self.lo_format = lo_format(split)
        self.range_flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self._plans = PlanBinder(dev, split)
        self.in_f32 = torch.zeros((B, H, W, 64), dtype=torch.float32, device=dev)         # channels 4..63 stay zero
        self.x_in = Operands((B, H, W, 64), dev, split)
        self.coarse, h, w = self._chain(list(net.coarse_net), self.x_in, H, W, final_f32=True)
        self.refine, h, w = self._chain(list(net.refine_conv_net), self.x_in, H, W, keep_last_f32=True)
        # self attention on [B, h, w, 128]: stacked 1x1 q / k / v convolution (16 + 16 + 128 = 160 output channels)
        att = net.refine_attn
        c = att.chanel_in
        if c != 128:
            raise LwbError("the attention kernel is specialised for SelfAttention(128)")
        wq = torch.cat([att.query_conv.weight, att.key_conv.weight, att.value_conv.weight], dim=0).detach().float()
        self.att_bias = torch.cat([att.query_conv.bias, att.key_conv.bias, att.value_conv.bias]).detach().float().contiguous()
        self.att_gamma = att.gamma.detach().float().contiguous()
        last = self.refine[-1]
        self.att_x = last["y_f32"]
        self.att = self._plans.conv(wq, last["out"].pair, B, h, w, pad=0, cout_pad=wq.shape[0], cin_pad=128)
        self.att_out = torch.empty((B, h, w, 128), dtype=torch.float32, device=dev)
        self.att_act = Operands((B, h, w, 128), dev, split)
        self.upsample, h, w = self._chain(list(net.refine_upsample_net), self.att_act, h, w, final_f32=True)
        self._plans.finalize()
        del self._plans

    def _chain(self, layers, x_act, h, w, final_f32=False, keep_last_f32=False):
        """Bind a Sequential of gated (de)conv layers.  -> (records, h, w) of the output."""
        B, dev, split = self.B, self.dev, self.split
        recs = []
        up_next = 1
        for i, m in enumerate(layers):
            is_de = isinstance(m, GatedDeConv2dWithActivation)
            g = m.conv2d if is_de else m
            conv = g.conv2d
            cout, cin, k, _ = conv.weight.shape
            stride, pad, dil = conv.stride[0], conv.padding[0], conv.dilation[0]
            cin_pad = x_act.hi.shape[3]
            wst = torch.cat([conv.weight, g.mask_conv2d.weight], dim=0).detach().float()
            cv = self._plans.conv(wst, x_act.pair, B, h, w, stride=stride, pad=pad, dil=dil, cout_pad=_ceil_to(2 * cout, 16),
                                  cin_pad=cin_pad)
            rec = dict(conv=cv, c=cout)
            rec["bias"] = torch.cat([conv.bias, g.mask_conv2d.bias]).detach().float().contiguous() if conv.bias is not None else None
            rec["act"] = 0 if g.activation is None else 2
            if g.batch_norm:
                bn = g.batch_norm2d
                rec["scale"], rec["shift"] = bn_affine(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
            else:
                rec["scale"] = rec["shift"] = None
            h, w = cv.desc.h_out, cv.desc.w_out
            last = (i == len(layers) - 1)
            # a GatedDeConv that FOLLOWS consumes this layer's output on the 2x nearest grid (networks/inpaintor.py:67)
            nxt_de = (not last) and isinstance(layers[i + 1], GatedDeConv2dWithActivation)
            rec["up"] = 2 if nxt_de else 1
            if last and final_f32:
                rec["out"], rec["y_f32"], rec["clamp"] = None, torch.empty((B, h, w, cout), dtype=torch.float32, device=dev), True
            else:
                rec["out"] = Operands((B, h * rec["up"], w * rec["up"], _ceil_to(cout, 64)), dev, split)
                rec["y_f32"] = torch.empty((B, h, w, cout), dtype=torch.float32, device=dev) if (last and keep_last_f32) else None
                rec["clamp"] = False
                x_act = rec["out"]
                h, w = h * rec["up"], w * rec["up"]
            recs.append(rec)
        return recs, h, w

    def _load(self, x):
        """NCHW fp32 [B,4,H,W] -> the shared 64-channel operand buffer (channels 4.. are zero)."""
        if tuple(x.shape) != (self.B, 4, self.H, self.W):
            raise LwbError("unexpected inpaintor input %s" % (tuple(x.shape),))
        self.in_f32[..., :4].copy_(x.permute(0, 2, 3, 1))
        K.norm_act_nhwc(self.in_f32, None, None, None, False, None, y_hi=self.x_in.hi, y_lo=self.x_in.lo,
                        lo_format=self.lo_format, range_flag=self.range_flag)

    def _run_chain(self, recs):
        for r in recs:
            r["conv"].plan.run()
            out = r["out"]
            K.gated_act_nhwc(r["conv"].out, r["c"], r["bias"], r["act"], r["scale"], r["shift"], upsample=r["up"], clamp=r["clamp"],
                             y_f32=r["y_f32"], y_hi=out.hi if out is not None else None, y_lo=out.lo if out is not None else None,
                             lo_format=self.lo_format, range_flag=self.range_flag)
        return recs[-1]

    def run_coarse(self, x):
        self.range_flag.zero_()
        self._load(x)
        last = self._run_chain(self.coarse)
        return K.nhwc_to_nchw(last["y_f32"])

    def run_refine(self, x):
        self._load(x)
        self._run_chain(self.refine)
        self.att.plan.run()
        K.self_attention_nhwc(self.att.out, self.att_bias, self.att_x, self.att_gamma, out=self.att_out)
        K.norm_act_nhwc(self.att_out, None, None, None, False, None, y_hi=self.att_act.hi, y_lo=self.att_act.lo,
                        lo_format=self.lo_format, range_flag=self.range_flag)
        last = self._run_chain(self.upsample)
        return K.nhwc_to_nchw(last["y_f32"])
