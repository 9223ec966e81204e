"""TEST INFRASTRUCTURE ONLY -- functional torch-fp32 restatement of torchvision's ``maskrcnn_resnet50_fpn`` in eval mode
(FrozenBatchNorm2d, the COCO configuration that utils/detectors.py:25-30 builds), without importing torchvision.

Follows torchvision 0.26 with its ``state_dict`` keys (current layout; impersonator_b200.detectors.remap_v1 converts
the published checkpoint's):
  GeneralizedRCNNTransform   normalise, bilinear resize (recompute_scale_factor), pad to a multiple of 32
  resnet50 + FPN             FrozenBN, maxpool 3x3 s2 p1, relu(bn3(conv3) + identity); laterals, nearest 2x top-down, P6
  RegionProposalNetwork      anchors (32..512, ratios .5/1/2, rounded), per-level top 1000, decode (1,1,1,1), clip,
                             small boxes < 1e-3, per-level NMS 0.7, first 1000
  RoIHeads                   MultiScaleRoIAlign 7x7 s2 (aligned=False), fc6/fc7, softmax, decode (10,10,5,5), > 0.05,
                             >= 1e-2, per-class NMS 0.5, top 100; mask RoIAlign 14x14, 4 convs, deconv, 1x1, sigmoid
  paste_masks_in_image       padding 1, expanded box truncated to int64, bilinear to the box size, clipped paste
Batched NMS is torchvision's vanilla branch (one greedy NMS per group), with NMS's own IoU arithmetic.
Pinned by tests/golden/make_maskrcnn_golden.py, which runs the reference's utils/detectors.py on torchvision with the
same synthetic weights and compares every stage.
"""
import math

import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
LAYERS = ((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2))      # planes, blocks, stride of the first block
ANCHOR_SIZES = (32, 64, 128, 256, 512)
ASPECT_RATIOS = (0.5, 1.0, 2.0)
CLIP = math.log(1000.0 / 16)
RPN_PRE_NMS, RPN_POST_NMS, RPN_NMS, RPN_MIN = 1000, 1000, 0.7, 1e-3
BOX_SCORE, BOX_NMS, BOX_MIN, BOX_DETS = 0.05, 0.5, 1e-2, 100

# ---- transform ---------------------------------------------------------------------------------------------------
def transform(img01):
    """[3,H,W] in [0,1] -> (padded [1,3,Hp,Wp], (h, w) after resize)."""
    mean = torch.tensor(MEAN, dtype=img01.dtype)
    std = torch.tensor(STD, dtype=img01.dtype)
    x = (img01 - mean[:, None, None]) / std[:, None, None]
    h, w = x.shape[-2:]
    scale = min(800.0 / min(h, w), 1333.0 / max(h, w))
    x = F.interpolate(x[None], scale_factor=scale, mode="bilinear", recompute_scale_factor=True, align_corners=False)[0]
    h2, w2 = x.shape[-2:]
    hp, wp = int(math.ceil(h2 / 32.0) * 32), int(math.ceil(w2 / 32.0) * 32)
    out = x.new_zeros((1, 3, hp, wp))
    out[0, :, :h2, :w2] = x
    return out, (h2, w2)


# ---- backbone ----------------------------------------------------------------------------------------------------
def frozen_bn(x, sd, p):
    scale = sd[p + ".weight"] * (sd[p + ".running_var"] + 1e-5).rsqrt()
    bias = sd[p + ".bias"] - sd[p + ".running_mean"] * scale
    return x * scale[None, :, None, None] + bias[None, :, None, None]


def bottleneck(x, sd, p, stride):
    o = F.relu(frozen_bn(F.conv2d(x, sd[p + ".conv1.weight"]), sd, p + ".bn1"))
    o = F.relu(frozen_bn(F.conv2d(o, sd[p + ".conv2.weight"], stride=stride, padding=1), sd, p + ".bn2"))
    o = frozen_bn(F.conv2d(o, sd[p + ".conv3.weight"]), sd, p + ".bn3")
    if (p + ".downsample.0.weight") in sd:
        x = frozen_bn(F.conv2d(x, sd[p + ".downsample.0.weight"], stride=stride), sd, p + ".downsample.1")
    return F.relu(o + x)


def body(x, sd, p="backbone.body"):
    x = F.relu(frozen_bn(F.conv2d(x, sd[p + ".conv1.weight"], stride=2, padding=3), sd, p + ".bn1"))
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    feats = []
    for li, (_, nblocks, stride) in enumerate(LAYERS):
        for bi in range(nblocks):
            x = bottleneck(x, sd, "%s.layer%d.%d" % (p, li + 1, bi), stride if bi == 0 else 1)
        feats.append(x)
    return feats


def fpn(feats, sd, p="backbone.fpn"):
    """C2..C5 -> (P2..P6, inner2..inner5)."""
    def inner(i, x):
        return F.conv2d(x, sd["%s.inner_blocks.%d.0.weight" % (p, i)], sd["%s.inner_blocks.%d.0.bias" % (p, i)])

    def layer(i, x):
        return F.conv2d(x, sd["%s.layer_blocks.%d.0.weight" % (p, i)], sd["%s.layer_blocks.%d.0.bias" % (p, i)], padding=1)

    last = inner(3, feats[3])
    inners = [last]
    results = [layer(3, last)]
    for i in range(2, -1, -1):
        lat = inner(i, feats[i])
        last = lat + F.interpolate(last, size=lat.shape[-2:], mode="nearest")
        inners.insert(0, last)
        results.insert(0, layer(i, last))
    results.append(F.max_pool2d(results[-1], 1, 2, 0))
    return results, inners


# ---- boxes -------------------------------------------------------------------------------------------------------
def cell_anchors(size):
    scales = torch.as_tensor([size], dtype=torch.float32)
    ratios = torch.as_tensor(ASPECT_RATIOS, dtype=torch.float32)
    h_ratios = torch.sqrt(ratios)
    w_ratios = 1 / h_ratios
    ws = (w_ratios[:, None] * scales[None, :]).view(-1)
    hs = (h_ratios[:, None] * scales[None, :]).view(-1)
    return (torch.stack([-ws, -hs, ws, hs], dim=1) / 2).round()


def anchors(grid, image_hw, size):
    """Anchors of one level, ordered (y, x, a).  Strides are image // grid (P6 at 800: 61)."""
    gh, gw = grid
    sh, sw = image_hw[0] // gh, image_hw[1] // gw
    sx = torch.arange(0, gw, dtype=torch.int32) * torch.tensor(sw, dtype=torch.int64)
    sy = torch.arange(0, gh, dtype=torch.int32) * torch.tensor(sh, dtype=torch.int64)
    yy, xx = torch.meshgrid(sy, sx, indexing="ij")
    xx, yy = xx.reshape(-1), yy.reshape(-1)
    shifts = torch.stack((xx, yy, xx, yy), dim=1)
    return (shifts.view(-1, 1, 4) + cell_anchors(size).view(1, -1, 4)).reshape(-1, 4)


def decode(rel, boxes, weights):
    """BoxCoder.decode_single: rel [N, 4k], boxes [N, 4] -> [N, k, 4]."""
    widths = boxes[:, 2] - boxes[:, 0]
    heights = boxes[:, 3] - boxes[:, 1]
    ctr_x = boxes[:, 0] + 0.5 * widths
    ctr_y = boxes[:, 1] + 0.5 * heights
    wx, wy, ww, wh = weights
    dx = rel[:, 0::4] / wx
    dy = rel[:, 1::4] / wy
    dw = torch.clamp(rel[:, 2::4] / ww, max=CLIP)
    dh = torch.clamp(rel[:, 3::4] / wh, max=CLIP)
    pcx = dx * widths[:, None] + ctr_x[:, None]
    pcy = dy * heights[:, None] + ctr_y[:, None]
    pw = torch.exp(dw) * widths[:, None]
    ph = torch.exp(dh) * heights[:, None]
    hw = torch.tensor(0.5, dtype=pcx.dtype) * pw
    hh = torch.tensor(0.5, dtype=pcy.dtype) * ph
    return torch.stack((pcx - hw, pcy - hh, pcx + hw, pcy + hh), dim=2)


def clip(boxes, hw):
    h, w = hw
    x = boxes[..., 0::2].clamp(min=0, max=w)
    y = boxes[..., 1::2].clamp(min=0, max=h)
    return torch.stack((x, y), dim=boxes.dim()).reshape(boxes.shape)


def small(boxes, min_size):
    ws, hs = boxes[:, 2] - boxes[:, 0], boxes[:, 3] - boxes[:, 1]
    return (ws >= min_size) & (hs >= min_size)


def nms(boxes, scores, thresh):
    """torchvision's CPU nms: stable descending sort, greedy, IoU = inter / (area_i + area_j - inter) > thresh."""
    if boxes.numel() == 0:
        return torch.zeros(0, dtype=torch.int64)
    order = torch.sort(scores, descending=True, stable=True)[1]
    b = boxes[order]
    x1, y1, x2, y2 = b.unbind(1)
    areas = (x2 - x1) * (y2 - y1)
    n = b.shape[0]
    sup = torch.zeros(n, dtype=torch.bool)
    keep = []
    for i in range(n):
        if sup[i]:
            continue
        keep.append(i)
        w = torch.clamp(torch.minimum(x2[i], x2[i + 1:]) - torch.maximum(x1[i], x1[i + 1:]), min=0)
        h = torch.clamp(torch.minimum(y2[i], y2[i + 1:]) - torch.maximum(y1[i], y1[i + 1:]), min=0)
        inter = w * h
        ovr = inter / (areas[i] + areas[i + 1:] - inter)
        sup[i + 1:] |= ovr > thresh
    return order[torch.tensor(keep, dtype=torch.int64)]


def batched_nms(boxes, scores, groups, thresh, stable=False):
    """torchvision's _batched_nms_vanilla.  Its final sort is torch's unstable one, so kept boxes of EQUAL score come
    out in an order only that call defines; ``stable=True`` orders them by index instead (what the CUDA sweep does)."""
    keep_mask = torch.zeros_like(scores, dtype=torch.bool)
    for g in torch.unique(groups):
        idx = torch.where(groups == g)[0]
        keep_mask[idx[nms(boxes[idx], scores[idx], thresh)]] = True
    keep = torch.where(keep_mask)[0]
    return keep[scores[keep].sort(descending=True, stable=stable)[1]]


# ---- RPN ---------------------------------------------------------------------------------------------------------
def rpn_head(P, sd, p="rpn.head"):
    """-> per level (logits [H*W*3], deltas [H*W*3, 4]) in (y, x, a) order."""
    out = []
    for x in P:
        t = F.relu(F.conv2d(x, sd[p + ".conv.0.0.weight"], sd[p + ".conv.0.0.bias"], padding=1))
        lg = F.conv2d(t, sd[p + ".cls_logits.weight"], sd[p + ".cls_logits.bias"])
        dl = F.conv2d(t, sd[p + ".bbox_pred.weight"], sd[p + ".bbox_pred.bias"])
        A, H, W = lg.shape[1:]
        out.append((lg.permute(0, 2, 3, 1).reshape(-1), dl.view(1, A, 4, H, W).permute(0, 3, 4, 1, 2).reshape(-1, 4)))
    return out


def topk(x, k):
    """Top k, descending, ties to the lower index."""
    k = min(k, x.numel())
    return torch.sort(x, descending=True, stable=True)[1][:k]


def rpn(P, image_hw, padded_hw, sd):
    """-> dict(levels=[dict(logits, deltas, top, proposals)], boxes [<=1000,4], scores)."""
    heads = rpn_head(P, sd)
    levels, cand_b, cand_s, cand_l = [], [], [], []
    for li, ((lg, dl), x) in enumerate(zip(heads, P)):
        anc = anchors(x.shape[-2:], padded_hw, ANCHOR_SIZES[li])
        top = topk(lg, RPN_PRE_NMS)
        props = decode(dl[top], anc[top], (1.0, 1.0, 1.0, 1.0))[:, 0]
        levels.append(dict(logits=lg, deltas=dl, top=top, proposals=props))
        cand_b.append(props)
        cand_s.append(lg[top])
        cand_l.append(torch.full((top.numel(),), li, dtype=torch.int64))
    boxes = clip(torch.cat(cand_b), image_hw)
    scores = torch.sigmoid(torch.cat(cand_s))
    lvl = torch.cat(cand_l)
    keep = torch.where(small(boxes, RPN_MIN))[0]
    keep = keep[scores[keep] >= 0.0]
    boxes, scores, lvl = boxes[keep], scores[keep], lvl[keep]
    k = batched_nms(boxes, scores, lvl, RPN_NMS)[:RPN_POST_NMS]
    return dict(levels=levels, candidates=(torch.cat(cand_b), torch.cat(cand_s), torch.cat(cand_l)),
                valid=keep, boxes=boxes[k], scores=scores[k])


# ---- RoI heads ---------------------------------------------------------------------------------------------------
def roi_levels(boxes):
    s = torch.sqrt((boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1]))
    lv = torch.floor(4 + torch.log2(s / 224) + torch.tensor(1e-6, dtype=s.dtype))
    return torch.clamp(lv, min=2, max=5).to(torch.int64) - 2


def roi_align(feat, boxes, out, scale, sampling=2):
    """torchvision roi_align (CPU arithmetic order), aligned=False: feat [1,C,H,W], boxes [R,4] -> [R,C,out,out]."""
    C, H, W = feat.shape[1:]
    R = boxes.shape[0]
    f = feat[0].reshape(C, H * W)
    sc = torch.tensor(scale, dtype=torch.float32)
    x1, y1, x2, y2 = (boxes[:, i] * sc for i in range(4))
    rw = torch.clamp(x2 - x1, min=1.0)
    rh = torch.clamp(y2 - y1, min=1.0)
    bw = rw / out
    bh = rh / out
    g = torch.tensor(float(sampling), dtype=torch.float32)
    acc = torch.zeros((R, C, out, out), dtype=torch.float32)
    ph = torch.arange(out, dtype=torch.float32)
    for iy in range(sampling):
        yy = (y1[:, None] + ph[None, :] * bh[:, None]) + (torch.tensor(iy + 0.5) * bh[:, None]) / g       # [R, out]
        for ix in range(sampling):
            xx = (x1[:, None] + ph[None, :] * bw[:, None]) + (torch.tensor(ix + 0.5) * bw[:, None]) / g
            Y = yy[:, :, None].expand(R, out, out)
            X = xx[:, None, :].expand(R, out, out)
            empty = (Y < -1.0) | (Y > H) | (X < -1.0) | (X > W)
            Y = torch.clamp(Y, min=0)
            X = torch.clamp(X, min=0)
            yl = Y.to(torch.int64)
            xl = X.to(torch.int64)
            ytop = yl >= H - 1
            xtop = xl >= W - 1
            yl = torch.where(ytop, H - 1, yl)
            xl = torch.where(xtop, W - 1, xl)
            Y = torch.where(ytop, yl.float(), Y)
            X = torch.where(xtop, xl.float(), X)
            yh = torch.where(ytop, yl, yl + 1)
            xh = torch.where(xtop, xl, xl + 1)
            ly, lx = Y - yl.float(), X - xl.float()
            hy, hx = 1.0 - ly, 1.0 - lx
            ws = [hy * hx, hy * lx, ly * hx, ly * lx]
            ps = [yl * W + xl, yl * W + xh, yh * W + xl, yh * W + xh]
            t = None                                    # output_val += w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4
            for wgt, pos in zip(ws, ps):
                wgt = torch.where(empty, 0.0, wgt)
                pos = torch.where(empty, 0, pos)
                v = f[:, pos.reshape(-1)].reshape(C, R, out, out).permute(1, 0, 2, 3)
                t = wgt[:, None] * v if t is None else t + wgt[:, None] * v
            acc = acc + t
    return acc / float(sampling * sampling)


def multiscale_roi_align(P, boxes, out):
    """MultiScaleRoIAlign over P2..P5 (scales 1/4 .. 1/32) -> ([R,256,out,out], levels)."""
    lv = roi_levels(boxes)
    res = torch.zeros((boxes.shape[0], P[0].shape[1], out, out), dtype=torch.float32)
    for l in range(4):
        idx = torch.where(lv == l)[0]
        if idx.numel():
            res[idx] = roi_align(P[l], boxes[idx], out, 2.0 ** -(l + 2))
    return res, lv


def box_head(feats, sd, p="roi_heads"):
    x = feats.flatten(1)
    x = F.relu(F.linear(x, sd[p + ".box_head.fc6.weight"], sd[p + ".box_head.fc6.bias"]))
    x = F.relu(F.linear(x, sd[p + ".box_head.fc7.weight"], sd[p + ".box_head.fc7.bias"]))
    return (F.linear(x, sd[p + ".box_predictor.cls_score.weight"], sd[p + ".box_predictor.cls_score.bias"]),
            F.linear(x, sd[p + ".box_predictor.bbox_pred.weight"], sd[p + ".box_predictor.bbox_pred.bias"]))


def postprocess_boxes(logits, regression, proposals, image_hw):
    """-> (boxes [D,4], scores [D], labels [D]) in the padded-image frame, plus the candidate tensors."""
    nc = logits.shape[-1]
    boxes = clip(decode(regression, proposals, (10.0, 10.0, 5.0, 5.0)), image_hw)
    scores = F.softmax(logits, -1)
    labels = torch.arange(nc).view(1, -1).expand_as(scores)
    boxes, scores, labels = boxes[:, 1:].reshape(-1, 4), scores[:, 1:].reshape(-1), labels[:, 1:].reshape(-1)
    inds = torch.where(scores > BOX_SCORE)[0]
    boxes, scores, labels = boxes[inds], scores[inds], labels[inds]
    keep = torch.where(small(boxes, BOX_MIN))[0]
    boxes, scores, labels = boxes[keep], scores[keep], labels[keep]
    keep = batched_nms(boxes, scores, labels, BOX_NMS)[:BOX_DETS]
    return boxes[keep], scores[keep], labels[keep], (boxes, scores, labels)


def mask_head(feats, labels, sd, p="roi_heads"):
    """[D,256,14,14] -> (logits of the label channel [D,28,28], probabilities)."""
    x = feats
    for i in range(4):
        x = F.relu(F.conv2d(x, sd["%s.mask_head.%d.0.weight" % (p, i)], sd["%s.mask_head.%d.0.bias" % (p, i)], padding=1))
    x = F.relu(F.conv_transpose2d(x, sd[p + ".mask_predictor.conv5_mask.weight"], sd[p + ".mask_predictor.conv5_mask.bias"], stride=2))
    lg = F.conv2d(x, sd[p + ".mask_predictor.mask_fcn_logits.weight"], sd[p + ".mask_predictor.mask_fcn_logits.bias"])
    lg = lg[torch.arange(lg.shape[0]), labels]
    return lg, lg.sigmoid()


def resize_boxes(boxes, from_hw, to_hw):
    rh = torch.tensor(to_hw[0], dtype=torch.float32) / torch.tensor(from_hw[0], dtype=torch.float32)
    rw = torch.tensor(to_hw[1], dtype=torch.float32) / torch.tensor(from_hw[1], dtype=torch.float32)
    x1, y1, x2, y2 = boxes.unbind(1)
    return torch.stack((x1 * rw, y1 * rh, x2 * rw, y2 * rh), dim=1)


def paste_masks(probs, boxes, hw, padding=1):
    """paste_masks_in_image: probs [D,M,M], boxes [D,4] (image frame) -> [D,1,H,W]."""
    M = probs.shape[-1]
    scale = float(M + 2 * padding) / M
    padded = F.pad(probs[:, None], (padding,) * 4)
    w_half = (boxes[:, 2] - boxes[:, 0]) * 0.5
    h_half = (boxes[:, 3] - boxes[:, 1]) * 0.5
    x_c = (boxes[:, 2] + boxes[:, 0]) * 0.5
    y_c = (boxes[:, 3] + boxes[:, 1]) * 0.5
    w_half = w_half * scale
    h_half = h_half * scale
    eb = torch.stack((x_c - w_half, y_c - h_half, x_c + w_half, y_c + h_half), dim=1).to(torch.int64)
    H, W = hw
    out = torch.zeros((probs.shape[0], 1, H, W), dtype=torch.float32)
    for i in range(probs.shape[0]):
        b = eb[i].tolist()
        w = max(int(b[2] - b[0] + 1), 1)
        h = max(int(b[3] - b[1] + 1), 1)
        m = F.interpolate(padded[i:i + 1], size=(h, w), mode="bilinear", align_corners=False)[0, 0]
        x0, x1 = max(b[0], 0), min(b[2] + 1, W)
        y0, y1 = max(b[1], 0), min(b[3] + 1, H)
        if x1 > x0 and y1 > y0:
            out[i, 0, y0:y1, x0:x1] = m[y0 - b[1]:y1 - b[1], x0 - b[0]:x1 - b[0]]
    return out


# ---- the whole model ---------------------------------------------------------------------------------------------
def forward(img01, sd):
    """MaskRCNN eval on one [3,H,W] image in [0,1] -> (detection dict like torchvision's, stage dict)."""
    x, image_hw = transform(img01)
    C = body(x, sd)
    P, inners = fpn(C, sd)
    r = rpn(P, image_hw, tuple(x.shape[-2:]), sd)
    props = r["boxes"]
    feats7, lv7 = multiscale_roi_align(P[:4], props, 7)
    logits, regression = box_head(feats7, sd)
    boxes, scores, labels, cand = postprocess_boxes(logits, regression, props, image_hw)
    feats14, lv14 = multiscale_roi_align(P[:4], boxes, 14)
    mlogits, mprobs = mask_head(feats14, labels, sd)
    orig = tuple(img01.shape[-2:])
    out_boxes = resize_boxes(boxes, image_hw, orig)
    masks = paste_masks(mprobs, out_boxes, orig)
    det = dict(boxes=out_boxes, labels=labels, scores=scores, masks=masks)
    st = dict(input=x, image_hw=image_hw, C=C, P=P, inners=inners, rpn=r, proposals=props, feats7=feats7, levels7=lv7,
              class_logits=logits, box_regression=regression, box_candidates=cand, det_boxes=boxes, feats14=feats14,
              levels14=lv14, mask_logits=mlogits, mask_probs=mprobs)
    return det, st


def person_id(labels, boxes, person=1):
    """PersonMaskRCNNDetector.get_bbox_max_ids: largest-area person (strict >, first wins), -1 if none."""
    pid, best = -1, -1
    for i in range(labels.shape[0]):
        if int(labels[i]) == person:
            x0, y0, x1, y1 = boxes[i]
            a = torch.abs((x1 - x0) * (y1 - y0))
            if a > best:
                best, pid = a, i
    return pid


def dilate(mask, ks):
    """utils/util.py:73-89 morph(mode='dilate'): [N,1,H,W] {0,1} -> {0,1}."""
    pad = ks // 2
    x = F.pad(mask, [pad, pad, pad, pad], value=0.0)
    return (F.conv2d(x, torch.ones(1, 1, ks, ks)) >= 1).float()


def inference(img, sd, ks=13, threshold=0.5):
    """PersonMaskRCNNDetector.inference: [3,S,S] in [-1,1] -> (box [4], mask [1,1,S,S], det, stages)."""
    det, st = forward((img + 1) / 2.0, sd)
    pid = person_id(det["labels"], det["boxes"])
    m = (det["masks"][pid] > threshold).float()
    if ks > 0:
        m = dilate(m[None], ks)
    return det["boxes"][pid], m, det, st
