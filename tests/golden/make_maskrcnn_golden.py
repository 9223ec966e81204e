"""Generates tests/golden/maskrcnn.npz -- run ONLY where the reference checkout and torchvision are installed (CPU).

Imports the REFERENCE ``utils/detectors.py`` unmodified, with ``torchvision.models.detection.maskrcnn_resnet50_fpn``
stubbed to return the FrozenBatchNorm2d build (what ``pretrained=True`` constructs) loaded with
impersonator_b200.synthetic.synthetic_maskrcnn_state(SEED) in the published checkpoint's key layout, and with
torchvision's batched NMS forced onto its vanilla branch (below 4000 box elements the CPU takes the coordinate-offset
branch, whose shifted boxes round IoUs differently).  Runs ``inference`` on synthetic_source(S) for S = 256 and 512,
checks the functional restatement oracle/maskrcnn_ref.py stage by stage against torchvision, and stores slices of
every stage (S = 256), the detections, chosen box and mask of both sizes, and the margin of every discrete decision
on the path to the chosen box and mask.  The source images themselves are pinned by their SHA-256 only.  Fails if a margin is
below 10x the GPU stage bar (2e-4 relative): then another seed must be picked (SEED = 21 passes)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")

import torchvision                                          # noqa: E402
from torchvision.models import resnet50                     # noqa: E402
from torchvision.models.detection import MaskRCNN          # noqa: E402
from torchvision.models.detection.backbone_utils import _resnet_fpn_extractor   # noqa: E402
from torchvision.ops import boxes as box_ops                # noqa: E402
from torchvision.ops.misc import FrozenBatchNorm2d          # noqa: E402

from impersonator_b200 import synthetic as S                # noqa: E402
from impersonator_b200.detectors import remap_v1            # noqa: E402
from oracle import maskrcnn_ref as R                        # noqa: E402

SEED = 21
BAR = 2e-4
SIZES = (256, 512)


def build_torchvision(sd_v1):
    backbone = _resnet_fpn_extractor(resnet50(weights=None, norm_layer=FrozenBatchNorm2d), 3)
    model = MaskRCNN(backbone, num_classes=91)
    model.load_state_dict(sd_v1)                           # version-1 keys: torchvision remaps them itself
    return model.eval()


def image_digest(img):
    """The source images are regenerated from their seed (synthetic_source); the golden pins them by digest."""
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(img.numpy()).tobytes()).hexdigest()


def rel(a, b):
    return float((a - b).abs().max() / max(b.abs().max(), 1e-12))


def iou(a, b):
    w = torch.clamp(torch.minimum(a[2], b[:, 2]) - torch.maximum(a[0], b[:, 0]), min=0)
    h = torch.clamp(torch.minimum(a[3], b[:, 3]) - torch.maximum(a[1], b[:, 1]), min=0)
    inter = w * h
    return inter / ((a[2] - a[0]) * (a[3] - a[1]) + (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1]) - inter)


def main():
    torch.set_grad_enabled(False)
    box_ops._batched_nms_coordinate_trick = box_ops._batched_nms_vanilla
    sd_v1 = S.synthetic_maskrcnn_state(SEED)
    sd = remap_v1(sd_v1)
    model = build_torchvision(sd_v1)
    torchvision.models.detection.maskrcnn_resnet50_fpn = lambda *a, **k: model
    from utils.detectors import PersonMaskRCNNDetector       # the reference
    ref = PersonMaskRCNNDetector(ks=13, threshold=0.5, to_gpu=False)
    out = dict(keys=np.array(sorted(sd_v1)), shapes=np.array([str(tuple(sd_v1[k].shape)) for k in sorted(sd_v1)]),
               keys_current=np.array(sorted(model.state_dict())), seed=np.array(SEED))
    for size in SIZES:
        img = S.synthetic_source(size)[0]
        box, mask = ref.inference(img)
        # torchvision, stage by stage
        images, _ = model.transform([(img + 1) / 2.0])
        feats = model.backbone(images.tensors)
        props, _ = model.rpn(images, feats)
        dets, _ = model.roi_heads(feats, props, images.image_sizes)
        # the restatement
        obox, omask, det, st = R.inference(img, sd, ks=13)
        P = list(feats.values())
        d = dict(input=rel(st["input"], images.tensors),
                 P=max(rel(a, b) for a, b in zip(st["P"], P)),
                 proposals=rel(st["proposals"], props[0]) if st["proposals"].shape == props[0].shape else float("inf"),
                 det_boxes=rel(st["det_boxes"], dets[0]["boxes"]) if st["det_boxes"].shape == dets[0]["boxes"].shape else float("inf"),
                 box=float((obox - box).abs().max()), mask=int((omask != mask).sum()))
        print("S=%d restatement vs torchvision:" % size, d, "detections", det["labels"].shape[0],
              "persons", int((det["labels"] == 1).sum()))
        assert d["input"] < 1e-6 and d["P"] < 1e-4 and d["proposals"] < 1e-5 and d["det_boxes"] < 1e-5
        assert d["box"] < 1e-4 and d["mask"] == 0
        # margins of the decisions on the path to the chosen box and mask
        pid = R.person_id(det["labels"], det["boxes"])
        areas = ((det["boxes"][:, 2] - det["boxes"][:, 0]) * (det["boxes"][:, 3] - det["boxes"][:, 1]))[det["labels"] == 1]
        top2 = torch.topk(areas, 2).values if areas.numel() >= 2 else torch.tensor([1.0, 0.0])
        cb, cs, cl = st["box_candidates"]
        same = (cl == det["labels"][pid]) & (cs > det["scores"][pid])
        ious = iou(st["det_boxes"][pid], cb[same])
        probs = st["mask_probs"][pid]
        margins = dict(score=float(det["scores"][pid] - R.BOX_SCORE),
                       iou=float((ious - R.BOX_NMS).abs().min()) if ious.numel() else 1.0,
                       area=float((top2[0] - top2[1]) / top2[0]),
                       mask_prob=float((probs - 0.5).abs().min()))
        print("S=%d margins" % size, margins)
        assert margins["score"] > 10 * BAR and margins["iou"] > 10 * BAR and margins["area"] > 10 * BAR
        r = st["rpn"]
        pre = "s%d_" % size
        near = (det["masks"][pid, 0] - 0.5).abs() < 1e-3          # pixels whose golden probability is within 1e-3 of 0.5
        out.update({
            pre + "img_sha256": np.array(image_digest(img)),
            pre + "det_boxes": det["boxes"].numpy(), pre + "det_scores": det["scores"].numpy(),
            pre + "det_labels": det["labels"].numpy().astype(np.int32),
            pre + "box": box.numpy(), pre + "mask_bits": np.packbits(mask.numpy().astype(bool)),
            pre + "near_half_bits": np.packbits(near.numpy()),
            pre + "pid": np.array(pid),
            pre + "margins": np.array([margins["score"], margins["iou"], margins["area"], margins["mask_prob"]]),
        })
        if size == SIZES[0]:                                       # stage slices, for the oracle's CPU check
            out.update({
                pre + "P_slices": np.concatenate([p[0, :2, ::4, ::4].reshape(-1).numpy() for p in st["P"]]),
                pre + "rpn_logits_head": np.concatenate([lv["logits"][:512].numpy() for lv in r["levels"]]),
                pre + "rpn_top": np.concatenate([lv["top"].numpy() for lv in r["levels"]]).astype(np.int32),
                pre + "rpn_deltas_head": np.concatenate([lv["deltas"][:128].numpy() for lv in r["levels"]]),
                pre + "rpn_proposals_head": np.concatenate([lv["proposals"][:128].numpy() for lv in r["levels"]]),
                pre + "proposals": st["proposals"].numpy(),
                pre + "class_logits_head": st["class_logits"][:128].numpy(),
                pre + "box_regression_head": st["box_regression"][:16].numpy(),
                pre + "mask_probs_head": st["mask_probs"][:8].numpy(),
            })
    np.savez_compressed(os.path.join(HERE, "maskrcnn.npz"), **out)
    print("wrote maskrcnn.npz (%.1f MB)" % (os.path.getsize(os.path.join(HERE, "maskrcnn.npz")) / 1e6))


if __name__ == "__main__":
    main()
