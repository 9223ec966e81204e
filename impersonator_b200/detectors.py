"""``PersonMaskRCNNDetector`` (utils/detectors.py:7-85) on this library's kernels.

The reference wraps torchvision's ``maskrcnn_resnet50_fpn(pretrained=True)`` (the COCO checkpoint with FrozenBatchNorm2d)
and keeps the largest person's mask.  Here ``.model`` is a ``MaskRCNN`` module with torchvision's ``state_dict`` keys
(the published checkpoint's version-1 names load too) whose children are parameter holders; ``forward`` drives

  transform: (x + 1) / 2, normalise, bilinear resize, pad to 32     lwb_det_transform
  stem 7x7 s2 + FrozenBN + ReLU + maxpool 3x3 s2 p1                 lwb_conv2d_direct_nchw, lwb_det_stem_pool
  ResNet-50 bottlenecks, FPN (laterals, top-down, 3x3), RPN conv    the wgmma conv engine in fp16x3 (FrozenBN folded
  and heads, fc6 / fc7 / predictors (1x1 convs over the RoIs),      into the weights), lwb_det_bias_act between convs,
  mask head convs, the 2x2 deconv (1x1 conv to 4 x 256 channels)    lwb_det_d2s_bias_relu after the deconv
  RPN top-k + decode + filters, batched NMS                         lwb_det_rpn, lwb_det_nms
  MultiScaleRoIAlign 7x7 / 14x14                                    lwb_det_roi_align (RoI-major NHWC)
  box post-processing, mask sigmoid, paste_masks_in_image           lwb_det_box_candidates + lwb_det_nms,
                                                                    lwb_det_mask_probs, lwb_det_paste_masks
  get_bbox_max_ids + threshold + morph(dilate)                      lwb_det_person_mask

Every intermediate lives in fixed-size device buffers with device-side counts; a forward pass synchronises once, to
read the number of detections.  The detector runs once per source image, so it always uses the fp16x3 operand mode
(its top-k, NMS and threshold decisions amplify operand error).  Weights are never downloaded: they come from
``weights=`` or from torch's hub cache, where ``pretrained=True`` leaves them.
"""
import math
import os

import numpy as np
import torch
import torch.nn as nn

from . import kernels as K
from ._lib import LwbError

WEIGHTS_FILE = "maskrcnn_resnet50_fpn_coco-bf2d0c1e.pth"
NUM_CLASSES = 91
LAYERS = ((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2))      # planes, blocks, stride of the first block
ANCHOR_SIZES = (32, 64, 128, 256, 512)
ASPECT_RATIOS = (0.5, 1.0, 2.0)
RPN_TOP, RPN_NMS, RPN_MIN = 1000, 0.7, 1e-3
BOX_SCORE, BOX_NMS, BOX_MIN, BOX_DETS = 0.05, 0.5, 1e-2, 100
XFORM_CLIP = math.log(1000.0 / 16)
SPLIT = 1                                                           # fp16x3


# ---- state_dict layouts ------------------------------------------------------------------------------------------
def remap_v1(sd):
    """The published checkpoint's version-1 key names -> torchvision's current ones (what its _load_from_state_dict
    does in rpn.py:54, mask_rcnn.py:317 and feature_pyramid_network.py:124).  Current keys pass through."""
    out = {}
    for k, v in sd.items():
        nk = k
        if k.startswith("rpn.head.conv.") and not k.startswith("rpn.head.conv.0.0."):
            nk = "rpn.head.conv.0.0." + k[len("rpn.head.conv."):]
        for blk in ("inner_blocks", "layer_blocks"):
            pre = "backbone.fpn.%s." % blk
            if k.startswith(pre):
                rest = k[len(pre):].split(".")
                if len(rest) == 2:
                    nk = pre + rest[0] + ".0." + rest[1]
        pre = "roi_heads.mask_head.mask_fcn"
        if k.startswith(pre):
            i, name = k[len(pre):].split(".", 1)
            nk = "roi_heads.mask_head.%d.0.%s" % (int(i) - 1, name)
        out[nk] = v
    return out


def to_v1(sd):
    """Current keys -> the published checkpoint's version-1 names (inverse of remap_v1)."""
    out = {}
    for k, v in sd.items():
        nk = k
        if k.startswith("rpn.head.conv.0.0."):
            nk = "rpn.head.conv." + k[len("rpn.head.conv.0.0."):]
        for blk in ("inner_blocks", "layer_blocks"):
            pre = "backbone.fpn.%s." % blk
            if k.startswith(pre):
                i, _, name = k[len(pre):].split(".")
                nk = pre + i + "." + name
        pre = "roi_heads.mask_head."
        if k.startswith(pre):
            i, _, name = k[len(pre):].split(".")
            nk = "roi_heads.mask_head.mask_fcn%d.%s" % (int(i) + 1, name)
        out[nk] = v
    return out


# ---- module tree (parameter holders with torchvision's names) -----------------------------------------------------
class FrozenBatchNorm2d(nn.Module):
    def __init__(self, n):
        super(FrozenBatchNorm2d, self).__init__()
        for name, val in (("weight", 1.0), ("bias", 0.0), ("running_mean", 0.0), ("running_var", 1.0)):
            self.register_buffer(name, torch.full((n,), val))

    def affine(self):
        """x * scale + shift, computed as torchvision's FrozenBatchNorm2d.forward does (eps 1e-5)."""
        scale = self.weight * (self.running_var + 1e-5).rsqrt()
        return scale, self.bias - self.running_mean * scale


def _conv(cin, cout, k, stride=1, bias=False):
    return nn.Conv2d(cin, cout, k, stride=stride, padding=k // 2, bias=bias)


class Bottleneck(nn.Module):
    def __init__(self, cin, planes, stride, down):
        super(Bottleneck, self).__init__()
        self.conv1, self.bn1 = _conv(cin, planes, 1), FrozenBatchNorm2d(planes)
        self.conv2, self.bn2 = _conv(planes, planes, 3, stride), FrozenBatchNorm2d(planes)
        self.conv3, self.bn3 = _conv(planes, planes * 4, 1), FrozenBatchNorm2d(planes * 4)
        self.stride = stride
        if down:
            self.downsample = nn.Sequential(_conv(cin, planes * 4, 1, stride), FrozenBatchNorm2d(planes * 4))


class ResNetBody(nn.Module):
    def __init__(self):
        super(ResNetBody, self).__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = FrozenBatchNorm2d(64)
        cin = 64
        for li, (planes, nb, stride) in enumerate(LAYERS):
            blocks = [Bottleneck(cin, planes, stride, True)] + [Bottleneck(planes * 4, planes, 1, False) for _ in range(nb - 1)]
            setattr(self, "layer%d" % (li + 1), nn.Sequential(*blocks))
            cin = planes * 4


class FeaturePyramidNetwork(nn.Module):
    def __init__(self):
        super(FeaturePyramidNetwork, self).__init__()
        self.inner_blocks = nn.ModuleList([nn.Sequential(_conv(c, 256, 1, bias=True)) for c in (256, 512, 1024, 2048)])
        self.layer_blocks = nn.ModuleList([nn.Sequential(_conv(256, 256, 3, bias=True)) for _ in range(4)])


class BackboneWithFPN(nn.Module):
    def __init__(self):
        super(BackboneWithFPN, self).__init__()
        self.body = ResNetBody()
        self.fpn = FeaturePyramidNetwork()


class RPNHead(nn.Module):
    def __init__(self):
        super(RPNHead, self).__init__()
        self.conv = nn.Sequential(nn.Sequential(_conv(256, 256, 3, bias=True)))
        self.cls_logits = _conv(256, 3, 1, bias=True)
        self.bbox_pred = _conv(256, 12, 1, bias=True)


class RegionProposalNetwork(nn.Module):
    def __init__(self):
        super(RegionProposalNetwork, self).__init__()
        self.head = RPNHead()


class RoIHeads(nn.Module):
    def __init__(self):
        super(RoIHeads, self).__init__()
        self.box_head = nn.Module()
        self.box_head.fc6 = nn.Linear(256 * 7 * 7, 1024)
        self.box_head.fc7 = nn.Linear(1024, 1024)
        self.box_predictor = nn.Module()
        self.box_predictor.cls_score = nn.Linear(1024, NUM_CLASSES)
        self.box_predictor.bbox_pred = nn.Linear(1024, NUM_CLASSES * 4)
        self.mask_head = nn.Sequential(*[nn.Sequential(_conv(256, 256, 3, bias=True)) for _ in range(4)])
        self.mask_predictor = nn.Module()
        self.mask_predictor.conv5_mask = nn.ConvTranspose2d(256, 256, 2, 2)
        self.mask_predictor.mask_fcn_logits = _conv(256, NUM_CLASSES, 1, bias=True)


def _pad_rows(w, b, rows):
    """Zero-pad a [cout, ...] weight and its bias to ``rows`` output channels (the conv engine's multiple of 16)."""
    wp = w.new_zeros((rows,) + tuple(w.shape[1:]))
    wp[:w.shape[0]] = w
    bp = b.new_zeros(rows)
    bp[:b.shape[0]] = b
    return wp, bp


class _Ops(object):
    """fp16 hi / lo conv operands with an optional fp32 copy."""
    __slots__ = ("hi", "lo", "f32")

    def __init__(self, shape, dev, f32=False):
        self.hi = torch.empty(shape, dtype=torch.float16, device=dev)
        self.lo = torch.empty(shape, dtype=torch.float16, device=dev)
        self.f32 = torch.empty(shape, dtype=torch.float32, device=dev) if f32 else None

    @property
    def pair(self):
        return (self.hi, self.lo)

    def out(self):
        return dict(y_f32=self.f32, y_hi=self.hi, y_lo=self.lo)


class _DetStream(object):
    """The detector bound to one input size: plans, buffers and folded weights."""

    def __init__(self, m, h, w, dev):
        self.dev, self.h, self.w = dev, h, w
        scale = min(800.0 / min(h, w), 1333.0 / max(h, w))
        self.ho, self.wo = int(math.floor(h * scale)), int(math.floor(w * scale))
        self.hp, self.wp = int(math.ceil(self.ho / 32.0) * 32), int(math.ceil(self.wo / 32.0) * 32)
        self.plans = []
        pend = []
        raws = {}

        def raw(n, hh, ww, c, tag=""):
            key = (n, hh, ww, c, tag)
            if key not in raws:
                raws[key] = torch.empty((n, hh, ww, c), dtype=torch.float32, device=dev)
            return raws[key]

        def plan(wt, x, n, hh, ww, stride=1, tag="", pad=None, out=None):
            cout, cin, kh, kw = wt.shape
            d = K.make_conv_desc(n, hh, ww, cin, cout, kh, kw, stride=stride, pad=kh // 2 if pad is None else pad, split=SPLIT)
            rec = dict(desc=d, x=x, w=wt, out=out if out is not None else raw(n, d.h_out, d.w_out, cout, tag))
            pend.append(rec)
            return rec

        def folded(conv, bn):
            sc, sh = bn.affine()
            return (conv.weight.detach().float() * sc[:, None, None, None]).contiguous(), sh.detach().float().contiguous()

        body = m.backbone.body
        self.w1 = body.conv1.weight.detach().float().contiguous()
        self.ss1 = tuple(t.detach().float().contiguous() for t in body.bn1.affine())
        hh, ww = self.hp // 4, self.wp // 4
        self.x0 = _Ops((1, hh, ww, 64), dev)
        x = self.x0
        self.blocks = []
        feats = []
        for li in range(4):
            layer = getattr(body, "layer%d" % (li + 1))
            for blk in layer:
                s = blk.stride
                planes = blk.conv1.weight.shape[0]
                ho, wo = (hh - 1) // s + 1, (ww - 1) // s + 1
                st = dict()
                w_, b_ = folded(blk.conv1, blk.bn1)
                st["c1"], st["b1"] = plan(w_, x.pair, 1, hh, ww), b_
                st["a1"] = _Ops((1, hh, ww, planes), dev)
                w_, b_ = folded(blk.conv2, blk.bn2)
                st["c2"], st["b2"] = plan(w_, st["a1"].pair, 1, hh, ww, stride=s), b_
                st["a2"] = _Ops((1, ho, wo, planes), dev)
                w_, b_ = folded(blk.conv3, blk.bn3)
                st["c3"] = plan(w_, st["a2"].pair, 1, ho, wo)
                if hasattr(blk, "downsample"):
                    wd, bd = folded(blk.downsample[0], blk.downsample[1])
                    st["ds"] = plan(wd, x.pair, 1, hh, ww, stride=s, tag="ds")
                    st["res"] = None
                    b_ = b_ + bd
                else:
                    st["ds"], st["res"] = None, x.f32
                st["b3"] = b_.contiguous()
                st["y"] = _Ops((1, ho, wo, planes * 4), dev, f32=True)
                x = st["y"]
                hh, ww = ho, wo
                self.blocks.append(st)
            feats.append(x)
        self.C = feats
        # FPN
        fpn = m.backbone.fpn
        self.fpn = []
        self.inners, self.P = [None] * 4, [None] * 5
        for i in range(3, -1, -1):
            c = feats[i]
            n_, h_, w_, _ = c.f32.shape
            inner, layer = fpn.inner_blocks[i][0], fpn.layer_blocks[i][0]
            lat = plan(inner.weight.detach().float().contiguous(), c.pair, 1, h_, w_, tag="lat")
            self.inners[i] = _Ops((1, h_, w_, 256), dev, f32=True)
            self.P[i] = _Ops((1, h_, w_, 256), dev, f32=True)
            lp = plan(layer.weight.detach().float().contiguous(), self.inners[i].pair, 1, h_, w_, tag="fpn")
            self.fpn.append(dict(i=i, lat=lat, lat_b=inner.bias.detach().float().contiguous(), layer=lp,
                                 layer_b=layer.bias.detach().float().contiguous()))
        h5, w5 = self.P[3].f32.shape[1:3]
        self.P[4] = _Ops((1, (h5 - 1) // 2 + 1, (w5 - 1) // 2 + 1, 256), dev, f32=True)
        # RPN
        head = m.rpn.head
        wc = head.conv[0][0]
        self.rpn_b = wc.bias.detach().float().contiguous()
        wh, bh = _pad_rows(torch.cat([head.cls_logits.weight, head.bbox_pred.weight]).detach().float(),
                           torch.cat([head.cls_logits.bias, head.bbox_pred.bias]).detach().float(), 16)
        self.rpn_head_b = bh.contiguous()
        self.rpn = []
        for l in range(5):
            _, gh, gw, _ = self.P[l].hi.shape
            t = _Ops((1, gh, gw, 256), dev)
            cp = plan(wc.weight.detach().float().contiguous(), self.P[l].pair, 1, gh, gw, tag="rpn")
            hp_ = plan(wh.contiguous(), t.pair, 1, gh, gw, tag="rpnhead")
            self.rpn.append(dict(conv=cp, t=t, head=hp_, grid=(gh, gw), stride=(self.hp // gh, self.wp // gw)))
        self.cells = torch.stack([_cell_anchors(s) for s in ANCHOR_SIZES])
        n_cand = sum(min(RPN_TOP, g["grid"][0] * g["grid"][1] * 3) for g in self.rpn)
        self.cand = dict(boxes=torch.zeros((n_cand, 4), dtype=torch.float32, device=dev),
                         scores=torch.zeros(n_cand, dtype=torch.float32, device=dev),
                         groups=torch.zeros(n_cand, dtype=torch.int32, device=dev),
                         valid=torch.zeros(n_cand, dtype=torch.int32, device=dev),
                         top=torch.zeros(n_cand, dtype=torch.int32, device=dev))
        # box head: the RoIs are the pixels of a [1, 125, 8] grid
        R = RPN_TOP
        self.R, self.rgrid = R, (R // 8, 8)
        rh_, rw_ = self.rgrid
        rh = m.roi_heads
        self.feats7 = _Ops((R, 7, 7, 256), dev, f32=True)
        self.levels7 = torch.zeros(R, dtype=torch.int32, device=dev)
        w6 = rh.box_head.fc6.weight.detach().float().view(1024, 256, 7, 7).permute(0, 2, 3, 1).reshape(1024, 12544, 1, 1)
        f7in = (self.feats7.hi.view(1, rh_, rw_, 12544), self.feats7.lo.view(1, rh_, rw_, 12544))
        self.fc6 = plan(w6.contiguous(), f7in, 1, rh_, rw_, tag="fc6")
        self.fc6_b = rh.box_head.fc6.bias.detach().float().contiguous()
        self.h6 = _Ops((1, rh_, rw_, 1024), dev)
        self.fc7 = plan(rh.box_head.fc7.weight.detach().float().view(1024, 1024, 1, 1).contiguous(), self.h6.pair, 1, rh_, rw_, tag="fc7")
        self.fc7_b = rh.box_head.fc7.bias.detach().float().contiguous()
        self.h7 = _Ops((1, rh_, rw_, 1024), dev)
        bp = rh.box_predictor
        wpr, bpr = _pad_rows(torch.cat([bp.cls_score.weight, bp.bbox_pred.weight]).detach().float(),
                             torch.cat([bp.cls_score.bias, bp.bbox_pred.bias]).detach().float(), 464)
        self.pred = plan(wpr.view(464, 1024, 1, 1).contiguous(), self.h7.pair, 1, rh_, rw_, tag="pred")
        self.pred_b = bpr.contiguous()
        self.pred_out = torch.empty((R, 464), dtype=torch.float32, device=dev)
        nslot = R * (NUM_CLASSES - 1)
        self.bcand = dict(boxes=torch.empty((nslot, 4), dtype=torch.float32, device=dev),
                          scores=torch.empty(nslot, dtype=torch.float32, device=dev),
                          groups=torch.empty(nslot, dtype=torch.int32, device=dev),
                          valid=torch.empty(nslot, dtype=torch.int32, device=dev))
        # mask head on the <= 100 detections
        D = BOX_DETS
        self.D = D
        self.feats14 = _Ops((D, 14, 14, 256), dev, f32=True)
        self.levels14 = torch.zeros(D, dtype=torch.int32, device=dev)
        self.mask_convs = []
        src = self.feats14
        for i in range(4):
            cv = rh.mask_head[i][0]
            dst = _Ops((D, 14, 14, 256), dev)
            self.mask_convs.append((plan(cv.weight.detach().float().contiguous(), src.pair, D, 14, 14, tag="mask%d" % (i % 2)),
                                    cv.bias.detach().float().contiguous(), dst))
            src = dst
        mp = m.roi_heads.mask_predictor
        wt = mp.conv5_mask.weight.detach().float().permute(2, 3, 1, 0).reshape(1024, 256, 1, 1)      # [(dy,dx,co), ci]
        self.deconv = plan(wt.contiguous(), src.pair, D, 14, 14, tag="deconv")
        self.deconv_b = mp.conv5_mask.bias.detach().float().contiguous()
        self.m28 = _Ops((D, 28, 28, 256), dev)
        wl, bl = _pad_rows(mp.mask_fcn_logits.weight.detach().float(), mp.mask_fcn_logits.bias.detach().float(), 96)
        self.mlog = plan(wl.contiguous(), self.m28.pair, D, 28, 28, tag="mlog")
        self.mlog_b = bl.contiguous()
        self.mask_logits = torch.empty((D, 28, 28), dtype=torch.float32, device=dev)
        self.mask_probs = torch.empty((D, 28, 28), dtype=torch.float32, device=dev)
        self.masks = torch.empty((D, 1, h, w), dtype=torch.float32, device=dev)
        self.out_boxes = torch.empty((D, 4), dtype=torch.float32, device=dev)
        # weights: one max|w| sync for the whole network, then the plans
        amax = torch.stack([p["w"].abs().max().float() for p in pend]).tolist()
        for p, a in zip(pend, amax):
            wp = K.pack_conv_weight(p["w"], split=SPLIT, absmax=a)
            p["plan"] = K.ConvPlan(p["desc"], p["x"], None, wp, p["out"], None)
            p["w"] = None
        self.ratio = (float(np.float32(h) / np.float32(self.ho)), float(np.float32(w) / np.float32(self.wo)))

    def run(self, img):
        """img [3,h,w] in [-1,1] -> device buffers (no host sync)."""
        self.x = K.det_transform(img, self.ho, self.wo, self.hp, self.wp)
        c1 = K.conv2d_direct_nchw(self.x, self.w1, None, stride=2, pad=3)
        K.det_stem_pool(c1, self.ss1[0], self.ss1[1], self.x0.hi, self.x0.lo)
        for st in self.blocks:
            st["c1"]["plan"].run()
            K.det_bias_act(st["c1"]["out"], st["b1"], relu=True, **st["a1"].out())
            st["c2"]["plan"].run()
            K.det_bias_act(st["c2"]["out"], st["b2"], relu=True, **st["a2"].out())
            st["c3"]["plan"].run()
            if st["ds"] is not None:
                st["ds"]["plan"].run()
            K.det_bias_act(st["c3"]["out"], st["b3"], relu=True, raw2=st["ds"]["out"] if st["ds"] is not None else None,
                           res=st["res"], **st["y"].out())
        for f in self.fpn:
            i = f["i"]
            f["lat"]["plan"].run()
            K.det_bias_act(f["lat"]["out"], f["lat_b"], res=self.inners[i + 1].f32 if i < 3 else None, res_half=True,
                           **self.inners[i].out())
            f["layer"]["plan"].run()
            K.det_bias_act(f["layer"]["out"], f["layer_b"], **self.P[i].out())
        K.det_bias_act(self.P[3].f32, None, step=2, out_hw=tuple(self.P[4].hi.shape[1:3]), **self.P[4].out())
        for r in self.rpn:
            r["conv"]["plan"].run()
            K.det_bias_act(r["conv"]["out"], self.rpn_b, relu=True, **r["t"].out())
            r["head"]["plan"].run()
        K.det_rpn([r["head"]["out"][0] for r in self.rpn], [r["stride"] for r in self.rpn], self.cells, self.rpn_head_b, RPN_TOP,
                  (self.ho, self.wo), RPN_MIN, XFORM_CLIP, self.cand)
        c = self.cand
        self.props = K.det_nms(c["boxes"], c["scores"], c["groups"], c["valid"], RPN_NMS, self.R)
        P4 = [p.f32 for p in self.P[:4]]
        K.det_roi_align(P4, self.props["boxes"], self.props["count"], 7, levels=self.levels7, **self.feats7.out())
        self.fc6["plan"].run()
        K.det_bias_act(self.fc6["out"], self.fc6_b, relu=True, **self.h6.out())
        self.fc7["plan"].run()
        K.det_bias_act(self.fc7["out"], self.fc7_b, relu=True, **self.h7.out())
        self.pred["plan"].run()
        K.det_bias_act(self.pred["out"], self.pred_b, y_f32=self.pred_out.view(self.pred["out"].shape))
        K.det_box_candidates(self.pred_out, NUM_CLASSES, self.props["boxes"], self.props["count"], (self.ho, self.wo), BOX_SCORE,
                             BOX_MIN, XFORM_CLIP, self.bcand)
        b = self.bcand
        self.dets = K.det_nms(b["boxes"], b["scores"], b["groups"], b["valid"], BOX_NMS, self.D, m_max=20 * self.R)
        K.det_roi_align(P4, self.dets["boxes"], self.dets["count"], 14, levels=self.levels14, **self.feats14.out())
        for pl, bias, dst in self.mask_convs:
            pl["plan"].run()
            K.det_bias_act(pl["out"], bias, relu=True, **dst.out())
        self.deconv["plan"].run()
        K.det_d2s_bias_relu(self.deconv["out"], self.deconv_b, y_hi=self.m28.hi, y_lo=self.m28.lo)
        self.mlog["plan"].run()
        K.det_mask_probs(self.mlog["out"], self.mlog_b, self.dets["groups"], self.dets["count"], self.mask_logits, self.mask_probs)
        K.det_paste_masks(self.mask_probs, self.dets["boxes"], self.dets["count"], self.ratio, (self.h, self.w), self.masks,
                          self.out_boxes)
        return self


def _cell_anchors(size):
    """AnchorGenerator.generate_anchors for one size and the three ratios, rounded (fp32, as torchvision)."""
    scales = torch.as_tensor([size], dtype=torch.float32)
    ratios = torch.as_tensor(ASPECT_RATIOS, dtype=torch.float32)
    h_ratios = torch.sqrt(ratios)
    w_ratios = 1 / h_ratios
    ws = (w_ratios[:, None] * scales[None, :]).view(-1)
    hs = (h_ratios[:, None] * scales[None, :]).view(-1)
    return (torch.stack([-ws, -hs, ws, hs], dim=1) / 2).round()


class MaskRCNN(nn.Module):
    """torchvision's MaskRCNN (resnet50_fpn, 91 classes) in eval mode: same ``state_dict`` keys, CUDA-only forward."""

    def __init__(self):
        super(MaskRCNN, self).__init__()
        self.backbone = BackboneWithFPN()
        self.rpn = RegionProposalNetwork()
        self.roi_heads = RoIHeads()
        self.__dict__['_lwb_streams'] = {}
        self.eval()

    def _invalidate(self):
        self.__dict__['_lwb_streams'] = {}

    def load_state_dict(self, state_dict, strict=True, **kw):
        sd = {k: v for k, v in remap_v1(state_dict).items() if not k.endswith("num_batches_tracked")}
        out = super(MaskRCNN, self).load_state_dict(sd, strict=strict, **kw)
        self._invalidate()
        return out

    def _apply(self, fn, *args, **kwargs):
        out = super(MaskRCNN, self)._apply(fn, *args, **kwargs)
        self._invalidate()
        return out

    def stream(self, h, w):
        dev = self.backbone.body.conv1.weight.device
        if dev.type != "cuda":
            raise LwbError("the Mask R-CNN detector runs on CUDA only (no CPU fallback): move it with .cuda()")
        streams = self.__dict__['_lwb_streams']
        if (h, w) not in streams:
            while len(streams) >= 2:
                streams.pop(next(iter(streams)))
            streams[(h, w)] = _DetStream(self, h, w, dev)
        return streams[(h, w)]

    def run(self, img):
        """img [3,h,w] in [-1,1] on the model's device -> the stream holding every stage (nothing synchronised)."""
        if img.dim() != 3 or img.shape[0] != 3:
            raise LwbError("the detector takes [3,H,W] images, got %s" % (tuple(img.shape),))
        st = self.stream(int(img.shape[1]), int(img.shape[2]))
        return st.run(img.float().contiguous())

    @torch.no_grad()
    def forward(self, images):
        """list of [3,H,W] in [0,1] -> [{'boxes', 'labels', 'scores', 'masks'}] like torchvision's eval output."""
        if self.training:
            raise LwbError("the detector runs in eval mode only")
        out = []
        for img in images:
            st = self.run(img * 2 - 1)
            n = int(st.dets["count"].item())
            out.append(dict(boxes=st.out_boxes[:n].clone(), labels=st.dets["groups"][:n].long(),
                            scores=st.dets["scores"][:n].clone(), masks=st.masks[:n].clone()))
        return out


def default_weights_path():
    return os.path.join(torch.hub.get_dir(), "checkpoints", WEIGHTS_FILE)


def load_weights(weights=None):
    """``weights``: a state dict, a path, or None for torch's hub cache.  Never downloads."""
    if isinstance(weights, dict):
        return weights
    path = weights if weights is not None else default_weights_path()
    if not os.path.exists(path):
        raise LwbError("Mask R-CNN weights not found at %s: place torchvision's %s there (this package never downloads)"
                       % (path, WEIGHTS_FILE))
    return torch.load(path, map_location="cpu", weights_only=True)


class PersonMaskRCNNDetector(object):
    """utils/detectors.py:7-85.  ``weights=`` is an extension (path or state dict); by default the COCO checkpoint is
    read from torch's hub cache."""
    PERSON_IDS = 1

    def __init__(self, ks=3, threshold=0.5, to_gpu=True, weights=None):
        self.model = MaskRCNN()
        self.model.load_state_dict(load_weights(weights))
        self.model.eval()
        self.threshold = threshold
        self.ks = ks
        if to_gpu:
            self.model = self.model.cuda()

    def forward(self, images):
        return self.model(images)

    def get_bbox_max_ids(self, labels, bboxs):
        """Largest-area person (strict >: the first of equal areas wins); -1 when there is none."""
        cur_pid = -1
        cur_bbox_area = -1
        for i, label in enumerate(labels):
            if label == self.PERSON_IDS:
                x0, y0, x1, y1 = bboxs[i]
                cur_area = torch.abs((x1 - x0) * (y1 - y0))
                if cur_area > cur_bbox_area:
                    cur_bbox_area = cur_area
                    cur_pid = i
        return cur_pid

    @torch.no_grad()
    def inference(self, img):
        """img [3,S,S] in [-1,1] -> (bbox [4], dilated body mask [1,1,S,S]).  pid = -1 (no person) takes the last
        detection, as the reference does; no detection at all raises LwbError."""
        st = self.model.run(img)
        _, box, mask = K.det_person_mask(st.out_boxes, st.dets["groups"], st.dets["count"], st.masks, self.threshold, self.ks,
                                         self.PERSON_IDS)
        if int(st.dets["count"].item()) == 0:
            raise LwbError("the detector found nothing in the source image")
        return box, mask
