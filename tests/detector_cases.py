"""Constructed inputs for the Mask R-CNN post-processing kernels (csrc/detect.cu), shared by the CPU tests, the GPU
tests and tests/golden/make_detector_cases_golden.py.

Every builder is seeded and returns plain CPU tensors in the layout the ``K.det_*`` wrapper takes.  The cases sit where
code like this goes wrong: ties across scan chunks, counts on 64-bit mask-word boundaries, IoU exactly at the
threshold, boxes outside the image or feature map, RoIs on a pyramid level boundary, ``count`` below the buffer size,
and nothing valid at all.

``oracle_*`` functions restate each kernel's contract with oracle/maskrcnn_ref.py, the torch-fp32 restatement that
tests/golden/detector_cases.npz pins to torchvision's own CPU ops.
"""
import math

import numpy as np
import torch

from oracle import maskrcnn_ref as R

F32 = np.float32
ANCHOR_SIZES = (32, 64, 128, 256, 512)


def f32(x):
    return float(np.float32(x))


def next_up(x, n=1):
    v = np.float32(x)
    for _ in range(n):
        v = np.nextafter(v, np.float32(np.inf), dtype=np.float32)
    return float(v)


def next_down(x, n=1):
    v = np.float32(x)
    for _ in range(n):
        v = np.nextafter(v, np.float32(-np.inf), dtype=np.float32)
    return float(v)


# ---- glue kernels ------------------------------------------------------------------------------------------------
TRANSFORM_HW = {"300": (300, 300), "511": (511, 511), "1024": (1024, 1024), "300x517": (300, 517), "777x420": (777, 420)}


def transform_cases():
    """Source images in [-1, 1]: smooth ramps plus noise, so that a resize off by a row or column shows."""
    out = {}
    for i, (name, (h, w)) in enumerate(TRANSFORM_HW.items()):
        rng = np.random.default_rng(900 + i)
        yy, xx = np.meshgrid(np.linspace(-1, 1, h), np.linspace(-1, 1, w), indexing="ij")
        img = np.stack([yy * 0.7, xx * 0.7, yy * xx * 0.7]) + rng.uniform(-0.3, 0.3, (3, h, w))
        out[name] = torch.from_numpy(img.astype(F32))
    return out


def detector_sizes(h, w):
    """(ho, wo, hp, wp) as impersonator_b200.detectors._DetStream derives them from the source size."""
    scale = min(800.0 / min(h, w), 1333.0 / max(h, w))
    ho, wo = int(math.floor(h * scale)), int(math.floor(w * scale))
    return ho, wo, int(math.ceil(ho / 32.0) * 32), int(math.ceil(wo / 32.0) * 32)


def glue_tensors(seed, *shapes, negative=False):
    rng = np.random.default_rng(seed)
    ts = [torch.from_numpy(rng.standard_normal(s).astype(F32)) for s in shapes]
    if negative:
        ts = [-(t.abs() + 0.01) for t in ts]
    return ts


# ---- RPN: top-k, decode (1, 1, 1, 1), clip, small-box filter, sigmoid ------------------------------------------------
def _rpn_case(grids, k, logits, deltas=None, stride=8, clip_hw=None, min_size=R.RPN_MIN, bias=None):
    """grids [(gh, gw)]; logits / deltas: per level [gh*gw*3] / [gh*gw*3, 4] (zeros when None); bias [16] (zeros)."""
    heads, strides = [], []
    for l, (gh, gw) in enumerate(grids):
        h = torch.zeros((gh, gw, 16))
        h[..., :3] = logits[l].view(gh, gw, 3)
        if deltas is not None:
            h[..., 3:15] = deltas[l].reshape(gh, gw, 12)
        heads.append(h)
        strides.append((stride * 2 ** l, stride * 2 ** l))
    if clip_hw is None:
        clip_hw = (grids[0][0] * stride, grids[0][1] * stride)
    cells = torch.stack([R.cell_anchors(s) for s in ANCHOR_SIZES])
    bias = torch.zeros(16) if bias is None else bias
    return dict(heads=heads, strides=strides, cells=cells, k=k, clip_hw=clip_hw, min_size=min_size, bias=bias)


def rpn_cases():
    rng = np.random.default_rng(101)
    C = {}

    def rnd(n, scale=1.0):
        return torch.from_numpy((rng.standard_normal(n) * scale).astype(F32))

    # n < k, n == k (k = 300: 9x10x3 = 270, 10x10x3 = 300), and n == k + 1 (k = 299)
    g = [(9, 10), (10, 10), (5, 4)]
    C["n_around_k"] = _rpn_case(g, 300, [rnd(a * b * 3) for a, b in g], [rnd((a * b * 3, 4), 0.2) for a, b in g])
    g = [(10, 10), (4, 3)]
    C["n_is_k_plus_1"] = _rpn_case(g, 299, [rnd(a * b * 3) for a, b in g], [rnd((a * b * 3, 4), 0.2) for a, b in g])
    # a full P2-size level whose logits take 3 values: 400 anchors at 2.0, every 7th of the rest at 0.5 (the 1000th
    # value, shared by ~17k anchors spread over every 1024-wide scan chunk), the others at -1
    n = 200 * 200 * 3
    lg = torch.full((n,), -1.0)
    lg[::7] = 0.5
    hi = torch.from_numpy(rng.choice(n, 400, replace=False))
    lg[hi] = 2.0
    C["p2_few_values"] = _rpn_case([(200, 200)], 1000, [lg], [rnd((n, 4), 0.1)], stride=4)
    g = [(40, 30)]
    C["all_equal"] = _rpn_case(g, 1000, [torch.full((3600,), 0.25)])
    # +0 / -0 alternating across the k boundary: 300 anchors at 1, 100 at -1, the other 800 at +-0.  The logit bias is
    # -0, the one bias that keeps both signs (+0 + -0 rounds to +0)
    n = 20 * 20 * 3
    lg = torch.zeros(n)
    lg[1::2] = -0.0
    perm = torch.from_numpy(rng.permutation(n))
    lg[perm[:300]] = 1.0
    lg[perm[300:400]] = -1.0
    C["signed_zero_tie"] = _rpn_case([(20, 20)], 1000, [lg], bias=torch.tensor([-0.0] * 3 + [0.0] * 13))
    # mixed signs, gh != gw, boxes decoded far outside the image (dx, dy of +-3 anchor widths)
    g = [(25, 40), (13, 20), (7, 10), (4, 5), (2, 3)]
    C["mixed_signs_outside"] = _rpn_case(g, 1000, [rnd(a * b * 3, 4.0) for a, b in g],
                                         [rnd((a * b * 3, 4), 1.5) for a, b in g])
    # dw / dh at XFORM_CLIP, one ulp above it, and far above it
    n = 8 * 8 * 3
    d = torch.zeros((n, 4))
    clip = f32(R.CLIP)
    vals = torch.tensor([clip, next_up(clip), next_down(clip), 10.0, -10.0, 0.0])
    d[:, 2] = vals[torch.arange(n) % 6]
    d[:, 3] = vals[(torch.arange(n) // 6) % 6]
    C["xform_clip"] = _rpn_case([(8, 8)], 1000, [rnd(n)], [d], stride=64)
    # widths exactly at RPN_MIN after clipping: the clip width is 1e-3f, so every box over x = 0 clips to width 1e-3f
    n = 10 * 10 * 3
    d = torch.zeros((n, 4))
    d[:, 0] = rnd(n, 0.5)
    C["min_width"] = _rpn_case([(10, 10)], 1000, [rnd(n)], [d], clip_hw=(80.0, f32(R.RPN_MIN)))
    return C


def oracle_rpn(case):
    """-> per-level list of dict(top, boxes (clipped), scores, valid)."""
    out = []
    for l, hd in enumerate(case["heads"]):
        gh, gw = hd.shape[:2]
        lg = (hd[..., :3] + case["bias"][:3]).reshape(-1)
        dl = (hd[..., 3:15] + case["bias"][3:15]).reshape(-1, 4)
        s = case["strides"][l]
        anc = R.anchors((gh, gw), (gh * s[0], gw * s[1]), ANCHOR_SIZES[l])
        top = R.topk(lg, case["k"])
        boxes = R.clip(R.decode(dl[top], anc[top], (1.0, 1.0, 1.0, 1.0))[:, 0], case["clip_hw"])
        scores = torch.sigmoid(lg[top])
        valid = R.small(boxes, case["min_size"]) & (scores >= 0.0)
        out.append(dict(top=top, boxes=boxes, scores=scores, valid=valid, anchors=anc[top], deltas=dl[top]))
    return out


# ---- batched NMS -------------------------------------------------------------------------------------------------
def _random_boxes(rng, n, extent=200.0, size=(4.0, 60.0)):
    xy = rng.uniform(0, extent, (n, 2))
    wh = rng.uniform(size[0], size[1], (n, 2))
    return torch.from_numpy(np.concatenate([xy, xy + wh], 1).astype(F32))


def _clustered_boxes(rng, n, clusters, jitter=3.0, size=(4.0, 60.0)):
    """Boxes jittered around a few centres, so that greedy NMS both keeps and suppresses."""
    base = _random_boxes(rng, clusters, size=size).numpy()
    pick = rng.integers(0, clusters, n)
    return torch.from_numpy((base[pick] + rng.uniform(-jitter, jitter, (n, 4))).astype(F32))


def _iou_pair(thresh):
    """Two nested boxes whose NMS IoU is exactly float32(thresh), and the first height above it that rounds the IoU
    above the threshold (computed with the oracle's own float32 arithmetic)."""
    t = np.float32(thresh)
    a = torch.tensor([[0.0, 0.0, 10.0, 10.0]])
    exact = torch.tensor([[0.0, 0.0, 10.0, 10.0 * float(t)]])
    assert float(_iou(a, exact)[0]) == float(t)
    h = float(exact[0, 3])
    while True:
        h = next_up(h)
        b = torch.tensor([[0.0, 0.0, 10.0, h]])
        if float(_iou(a, b)[0]) > float(t):
            return a[0], exact[0], b[0]


def _iou(a, b):
    """The NMS kernel's IoU (torchvision nms_kernel.cpp order), float32."""
    w = torch.clamp(torch.minimum(a[:, 2], b[:, 2]) - torch.maximum(a[:, 0], b[:, 0]), min=0)
    h = torch.clamp(torch.minimum(a[:, 3], b[:, 3]) - torch.maximum(a[:, 1], b[:, 1]), min=0)
    inter = w * h
    return inter / ((a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1]) + (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1]) - inter)


def _nms_case(boxes, scores, groups, valid=None, thresh=0.5, max_keep=None, m_max=None):
    n = boxes.shape[0]
    return dict(boxes=boxes.float().contiguous(), scores=scores.float().contiguous(), groups=groups.int().contiguous(),
                valid=None if valid is None else valid.int().contiguous(), thresh=thresh,
                max_keep=max_keep or n, m_max=m_max or n)


def nms_cases():
    rng = np.random.default_rng(202)
    C = {}
    # valid counts at the 64-bit mask-word and 64-box block boundaries
    for m in (1, 63, 64, 65, 127, 128, 129, 4097):
        b = _clustered_boxes(rng, m, max(1, m // 6))
        s = torch.from_numpy(rng.uniform(0, 1, m).astype(F32))
        C["count_%d" % m] = _nms_case(b, s, torch.zeros(m), thresh=0.5)
    # IoU exactly at 0.5 and 0.7f (kept: suppression is strict >) and the next representable IoU above (suppressed)
    for t in (0.5, 0.7):
        a, exact, above = _iou_pair(t)
        boxes, groups = [], []
        for g in range(3):
            off = torch.tensor([40.0 * g, 0.0, 40.0 * g, 0.0])
            boxes += [a + off, exact + off, above + off]
            groups += [g] * 3
        boxes = torch.stack(boxes)
        # the big box first; then within each group the exact pair is kept and the above one is suppressed
        s = torch.tensor([0.9, 0.8, 0.7] * 3)
        C["iou_at_%g" % t] = _nms_case(boxes, s, torch.tensor(groups), thresh=t)
    # identical, nested and zero-area boxes (0 / 0 IoU never suppresses)
    boxes = torch.tensor([[10, 10, 50, 50]] * 3 + [[12, 12, 48, 48], [0, 0, 100, 100], [20, 20, 30, 30]]
                         + [[5, 5, 5, 5]] * 3 + [[7, 7, 7, 20], [7, 7, 20, 7]], dtype=torch.float32)
    s = torch.from_numpy(rng.uniform(0, 1, boxes.shape[0]).astype(F32))
    C["identical_nested_zero_area"] = _nms_case(boxes, s, torch.zeros(boxes.shape[0]), thresh=0.5)
    # equal scores within a group and across groups (ties to the lower slot)
    b = _clustered_boxes(rng, 300, 20)
    s = torch.from_numpy(rng.choice(np.array([0.25, 0.5, 0.75], F32), 300))
    C["equal_scores"] = _nms_case(b, s, torch.from_numpy(rng.integers(0, 3, 300)), thresh=0.5)
    # 90 interleaved groups, sparse valid
    n = 2000
    b = _clustered_boxes(rng, n, 40, jitter=6.0)
    s = torch.from_numpy(rng.uniform(0, 1, n).astype(F32))
    v = torch.from_numpy(rng.uniform(0, 1, n) < 0.3)
    C["groups_90_sparse"] = _nms_case(b, s, torch.arange(n) % 90 + 1, valid=v, thresh=0.5)
    # nothing valid: count 0, keep all -1
    C["none_valid"] = _nms_case(b[:200], s[:200], torch.zeros(200), valid=torch.zeros(200), thresh=0.7, max_keep=50)
    # max_keep below the number of survivors
    C["max_keep_cut"] = _nms_case(b[:1000], s[:1000], torch.arange(1000) % 5, thresh=0.7, max_keep=37)
    # RPN scale (5 levels, ~4.5k candidates, IoU 0.7, first 1000) and box-stage scale (R x 90 slots, IoU 0.5, top 100)
    for seed in (0, 1, 2):
        r = np.random.default_rng(300 + seed)
        n = 4500
        b = _clustered_boxes(r, n, 150, jitter=5.0, size=(40.0, 150.0))
        s = torch.from_numpy(r.uniform(0, 1, n).astype(F32))
        v = torch.from_numpy(r.uniform(0, 1, n) < 0.95)
        C["rpn_scale_%d" % seed] = _nms_case(b, s, torch.from_numpy(r.integers(0, 5, n)), valid=v, thresh=0.7, max_keep=1000)
        n = 1000 * 90
        b = _clustered_boxes(r, n, 20, jitter=8.0, size=(40.0, 150.0))
        s = torch.from_numpy(r.uniform(0, 1, n).astype(F32))
        v = torch.from_numpy(r.uniform(0, 1, n) < 0.04)
        C["box_scale_%d" % seed] = _nms_case(b, s, torch.arange(n) % 90 + 1, valid=v, thresh=0.5, max_keep=100, m_max=20000)
    return C


def oracle_nms(case):
    """-> keep (slot indices, descending score, ties by slot), truncated to max_keep."""
    n = case["scores"].shape[0]
    vi = torch.arange(n) if case["valid"] is None else torch.where(case["valid"] != 0)[0]
    keep = vi[R.batched_nms(case["boxes"][vi], case["scores"][vi], case["groups"][vi].long(), case["thresh"], stable=True)]
    return keep[:case["max_keep"]]


# ---- MultiScaleRoIAlign ------------------------------------------------------------------------------------------
PYRAMID_HW = ((50, 38), (25, 19), (13, 10), (7, 5))          # non-square; the image is 200 x 152
ROI_IMAGE_HW = (200, 152)
ROI_C = 8


def roi_pyramid(seed=404):
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.standard_normal((1, ROI_C, h, w)).astype(F32)) for h, w in PYRAMID_HW]


def roi_boxes():
    """-> (boxes [r_max, 4], count).  Rows past ``count`` hold boxes the kernel must not use."""
    rows = []
    # sqrt(area) within +-64 ulps of the level boundaries 112, 224, 448 (squares, and 2:1 boxes of the same area)
    for s0 in (112.0, 224.0, 448.0):
        for k in range(-64, 65, 4):
            s = next_up(s0, k) if k >= 0 else next_down(s0, -k)
            rows.append([3.0, 5.0, 3.0 + s, 5.0 + s])
            rows.append([1.0, 2.0, 1.0 + f32(s * math.sqrt(2)), 2.0 + f32(s / math.sqrt(2))])
    # zero-area and very large boxes
    rows += [[20, 20, 20, 20], [0, 0, 0, 0], [-50, -50, 4000, 3000], [0, 0, 1e4, 1e4]]
    # level-0 boxes (14 feature cells = 56 px) whose sample points land exactly on -1, 0, H-1, H and beyond H
    # (bin height 2 feature cells: samples at y1 + 0.5 + j, j = 0..13)
    H, W = PYRAMID_HW[0]
    for y1 in (-1.5, -0.5, H - 13.5, H - 12.5, H - 10.0):
        for x1 in (-1.5, W - 13.5, W - 12.5):
            rows.append([4 * x1, 4 * y1, 4 * (x1 + 14), 4 * (y1 + 14)])
    # boxes smaller than one feature cell (rw, rh clamped to 1)
    rows += [[30.0, 40.0, 31.0, 40.5], [100.0, 7.0, 102.5, 9.0], [60.0, 60.0, 60.25, 64.0]]
    count = len(rows)
    rows += [[1.0, 1.0, 30.0, 30.0], [10.0, 10.0, 150.0, 150.0], [0.0, 0.0, 5.0, 5.0]]       # beyond count
    return torch.tensor(rows, dtype=torch.float32), count


def oracle_roi_align(P, boxes, count, out):
    """-> (features [r_max, out, out, C] NHWC, zero past count; levels [count])."""
    f, lv = R.multiscale_roi_align(P, boxes[:count], out)
    y = torch.zeros((boxes.shape[0], out, out, P[0].shape[1]))
    y[:count] = f.permute(0, 2, 3, 1)
    return y, lv


# ---- box candidates (softmax, decode (10, 10, 5, 5), clip, > 0.05, >= 1e-2) --------------------------------------
NC, PRED_LD = 91, 464


def box_candidate_cases():
    rng = np.random.default_rng(505)
    C = {}
    r_max = 48
    lg = np.zeros((r_max, NC), F32)
    kinds = []
    for r in range(r_max):
        kind = r % 6
        kinds.append(kind)
        if kind == 0:                                   # one dominant class
            lg[r] = rng.standard_normal(NC) * 0.5
            lg[r, rng.integers(1, NC)] = 9.0
        elif kind == 1:                                 # flat: 1/91 < 0.05, nothing valid
            lg[r] = 1.5
        elif kind == 2:                                 # exactly 19 classes at 0.0521 > 0.05, the most a row can hold
            lg[r] = 0.0
            lg[r, rng.choice(np.arange(1, NC), 19, replace=False)] = 6.0
        elif kind == 3:                                 # logits of +-80
            lg[r] = -80.0
            lg[r, rng.integers(0, NC)] = 80.0
            lg[r, rng.integers(1, NC)] = 80.0
        else:                                           # random
            lg[r] = rng.standard_normal(NC) * 3.0
    deltas = (rng.standard_normal((r_max, NC, 4)) * 0.5).astype(F32)
    clip = np.float32(5.0 * np.float32(R.CLIP))
    big = np.array([clip, np.nextafter(clip, np.float32(np.inf)), 40.0, -40.0], F32)
    deltas[5::6, :, 2] = big[np.arange(NC) % 4]          # dw, dh at, above and far beyond the clip (weights 5)
    deltas[5::6, :, 3] = big[(np.arange(NC) // 4) % 4]
    deltas[4::12, :, :2] = rng.standard_normal((len(range(4, r_max, 12)), NC, 2)).astype(F32) * 80.0    # far outside
    props = _random_boxes(rng, r_max, extent=300.0, size=(2.0, 200.0))
    C["mixed"] = _box_case(lg, deltas, props, count=41, clip_hw=(320.0, 352.0))
    # widths exactly at BOX_MIN: the clip width is 1e-2f
    lg2 = np.zeros((16, NC), F32)
    lg2[:, 1:11] = 5.0
    d2 = (rng.standard_normal((16, NC, 4)) * 0.5).astype(F32)
    C["min_width"] = _box_case(lg2, d2, _random_boxes(rng, 16, extent=5.0), count=16, clip_hw=(100.0, f32(R.BOX_MIN)))
    return C


def _box_case(lg, deltas, props, count, clip_hw):
    r_max = lg.shape[0]
    pred = torch.zeros((r_max, PRED_LD))
    pred[:, :NC] = torch.from_numpy(lg)
    pred[:, NC:NC * 5] = torch.from_numpy(deltas.reshape(r_max, NC * 4))
    return dict(pred=pred, props=props.contiguous(), count=count, clip_hw=clip_hw)


def oracle_box_candidates(case):
    """-> slot-major (boxes [R*90, 4], scores [R*90], groups, valid) in the kernel's (RoI, class) order."""
    pred, props = case["pred"], case["props"]
    r_max = pred.shape[0]
    lg, reg = pred[:, :NC], pred[:, NC:NC * 5]
    boxes = R.clip(R.decode(reg, props, (10.0, 10.0, 5.0, 5.0)), case["clip_hw"])[:, 1:].reshape(-1, 4)
    scores = torch.softmax(lg, -1)[:, 1:].reshape(-1)
    groups = torch.arange(1, NC).repeat(r_max)
    live = (torch.arange(r_max) < case["count"]).repeat_interleave(NC - 1)
    valid = live & (scores > R.BOX_SCORE) & R.small(boxes, R.BOX_MIN)
    return boxes, scores, groups, valid


# ---- mask probabilities, paste, person pick ------------------------------------------------------------------------
def mask_probs_case():
    rng = np.random.default_rng(606)
    d_max, ld = 6, 96
    raw = torch.from_numpy((rng.standard_normal((d_max, 28, 28, ld)) * 4).astype(F32))
    bias = torch.from_numpy(rng.standard_normal(ld).astype(F32))
    labels = torch.tensor([1, 90, 1, 90, 7, 3], dtype=torch.int32)
    return dict(raw=raw, bias=bias, labels=labels, count=4)


def oracle_mask_probs(case):
    raw, lab, n = case["raw"], case["labels"].long(), case["count"]
    lg = torch.zeros(raw.shape[:3])
    lg[:n] = raw[torch.arange(n), :, :, lab[:n]] + case["bias"][lab[:n]][:, None, None]
    p = torch.zeros_like(lg)
    p[:n] = torch.sigmoid(lg[:n])
    return lg, p


def paste_cases():
    rng = np.random.default_rng(707)
    C = {}

    def probs(d, m=28):
        return torch.from_numpy(rng.uniform(0, 1, (d, m, m)).astype(F32))

    # boxes in the detection frame (ho x wo), pasted into an h x w image
    boxes = torch.tensor([
        [10.0, 20.0, 200.0, 300.0],         # inside
        [-40.0, -30.0, 60.0, 90.0],         # partly outside, negative expanded corners (truncate toward zero)
        [-3.7, -2.2, 2.9, 4.1],             # straddles 0: -0.x corners truncate to 0, not -1
        [700.0, 500.0, 900.0, 700.0],       # wholly outside
        [100.0, 100.0, 100.4, 100.3],       # sub-pixel
        [-200.0, -150.0, 1100.0, 1000.0],   # larger than the image
        [50.0, 60.0, 52.0, 300.0],          # thin
        [5.0, 5.0, 400.0, 400.0],           # past count
    ])
    C["square_300"] = dict(probs=probs(8), boxes=boxes, count=7, from_hw=(800, 800), to_hw=(300, 300))
    C["non_square"] = dict(probs=probs(8), boxes=boxes, count=8, from_hw=(800, 1088), to_hw=(256, 348))
    C["dyadic_512"] = dict(probs=probs(8), boxes=boxes, count=5, from_hw=(800, 800), to_hw=(512, 512))
    return C


def paste_ratio(case):
    (fh, fw), (th, tw) = case["from_hw"], case["to_hw"]
    return float(np.float32(th) / np.float32(fh)), float(np.float32(tw) / np.float32(fw))


def oracle_paste(case):
    """-> (masks [d_max, 1, h, w], zero past count; resized boxes [d_max, 4], zero past count)."""
    n = case["count"]
    ob = R.resize_boxes(case["boxes"][:n], case["from_hw"], case["to_hw"])
    m = torch.zeros((case["boxes"].shape[0], 1) + tuple(case["to_hw"]))
    m[:n] = R.paste_masks(case["probs"][:n], ob, case["to_hw"])
    b = torch.zeros_like(case["boxes"])
    b[:n] = ob
    return m, b


def person_cases():
    rng = np.random.default_rng(808)
    H, W = 40, 36
    boxes = torch.tensor([[0, 0, 10, 10], [30, 0, 10, 20], [5, 5, 25, 15], [0, 0, 20, 10], [2, 2, 3, 3],
                          [0, 0, 10, 20]], dtype=torch.float32)       # row 1: negative width, signed area -400
    masks = torch.from_numpy(rng.choice(np.array([0.1, 0.5, 0.9], F32), (6, 1, H, W), p=[0.9, 0.07, 0.03]))
    masks[:, :, ::9, ::7] = 0.5                                      # exactly at the threshold: not > 0.5
    C = {}
    C["largest_negative_width"] = dict(boxes=boxes, labels=torch.tensor([1, 1, 3, 1, 1, 2]), count=6, masks=masks)
    C["equal_areas_first_wins"] = dict(boxes=boxes, labels=torch.tensor([3, 3, 2, 1, 1, 1]), count=6, masks=masks)
    # the only person sits past count: no person, so the last live detection
    C["no_person_last"] = dict(boxes=boxes, labels=torch.tensor([3, 2, 5, 7, 9, 1]), count=5, masks=masks)
    C["count_0"] = dict(boxes=boxes, labels=torch.tensor([1, 1, 1, 1, 1, 1]), count=0, masks=masks)
    return C


def oracle_person(case, ks, thresh=0.5):
    """-> (pid, box, mask [1, 1, h, w]).  No person: the last detection; count 0: pid -1 and zeros."""
    n = case["count"]
    H, W = case["masks"].shape[-2:]
    if n == 0:
        return -1, torch.zeros(4), torch.zeros((1, 1, H, W))
    pid = R.person_id(case["labels"][:n], case["boxes"][:n])
    pid = pid if pid >= 0 else n - 1
    m = (case["masks"][pid:pid + 1] > thresh).float()
    if ks > 0:
        m = R.dilate(m, ks)
    return pid, case["boxes"][pid], m
