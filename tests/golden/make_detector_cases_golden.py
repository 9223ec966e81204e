"""Generates tests/golden/detector_cases.npz -- run where torchvision 0.26 is installed (CPU).

Runs the constructed cases of tests/detector_cases.py through torchvision's own CPU ops: ``ops.batched_nms`` (forced
onto its vanilla branch, one greedy NMS per group, as make_maskrcnn_golden.py does), ``MultiScaleRoIAlign`` with its
``LevelMapper``, ``BoxCoder.decode``, ``clip_boxes_to_image``, ``remove_small_boxes``, ``resize_boxes``,
``paste_masks_in_image`` and ``GeneralizedRCNNTransform``'s normalise + resize.  It stores keep lists, levels and valid
flags whole and float outputs sub-sampled.  tests/test_detector_kernels_cpu.py checks that oracle/maskrcnn_ref.py
reproduces every one of them; the GPU tests then hold the kernels to that oracle.

torchvision's batched NMS returns kept boxes of EQUAL score in the order of an unstable sort; the golden stores them by
(score descending, slot ascending), after checking that this is a reordering among equal scores only.

The archive is written with fixed zip timestamps, so rerunning the script reproduces it byte for byte."""
import io
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import torchvision                                                      # noqa: E402
from torchvision.models.detection import _utils as det_utils            # noqa: E402
from torchvision.models.detection.roi_heads import paste_masks_in_image   # noqa: E402
from torchvision.models.detection.transform import GeneralizedRCNNTransform, resize_boxes   # noqa: E402
from torchvision.ops import MultiScaleRoIAlign, boxes as box_ops       # noqa: E402

import detector_cases as DC                                             # noqa: E402
from oracle import maskrcnn_ref as R                                    # noqa: E402

OUT = os.path.join(HERE, "detector_cases.npz")


def save_npz(path, arrays):
    """np.savez_compressed with a fixed member timestamp and order."""
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            b = io.BytesIO()
            np.lib.format.write_array(b, np.ascontiguousarray(arrays[k]), allow_pickle=False)
            z.writestr(info, b.getvalue())
    with open(path, "wb") as f:
        f.write(buf.getvalue())


def tv_batched_nms(boxes, scores, groups, thresh):
    keep = torchvision.ops.batched_nms(boxes, scores, groups, thresh)
    canon = keep.sort().values
    canon = canon[scores[canon].sort(descending=True, stable=True)[1]]
    assert torch.equal(scores[keep], scores[canon])                   # differs only among equal scores
    return canon


def main():
    torch.set_grad_enabled(False)
    torch.set_num_threads(1)
    assert torchvision.__version__.startswith("0.26"), torchvision.__version__
    box_ops._batched_nms_coordinate_trick = box_ops._batched_nms_vanilla
    out = {}
    # RPN: top-k (stable sort), decode (1, 1, 1, 1), clip, small boxes
    coder = det_utils.BoxCoder(weights=(1.0, 1.0, 1.0, 1.0))
    for name, case in DC.rpn_cases().items():
        for l, o in enumerate(DC.oracle_rpn(case)):
            p = "rpn/%s/%d/" % (name, l)
            b = coder.decode(o["deltas"], [o["anchors"]])[:, 0]
            b = box_ops.clip_boxes_to_image(b, case["clip_hw"])
            keep = box_ops.remove_small_boxes(b, case["min_size"])
            valid = torch.zeros(b.shape[0], dtype=torch.bool)
            valid[keep] = True
            out[p + "top"] = o["top"].numpy().astype(np.int32)
            out[p + "valid"] = valid.numpy()
            out[p + "boxes"] = b[::7].numpy()
            print("rpn %-20s level %d: n %6d, valid %4d / %4d" % (name, l, case["heads"][l].shape[0] * case["heads"][l].shape[1] * 3,
                                                              int(valid.sum()), valid.numel()))
    # NMS
    for name, case in DC.nms_cases().items():
        n = case["scores"].shape[0]
        vi = torch.arange(n) if case["valid"] is None else torch.where(case["valid"] != 0)[0]
        keep = vi[tv_batched_nms(case["boxes"][vi], case["scores"][vi], case["groups"][vi].long(), case["thresh"])]
        out["nms/%s/keep" % name] = keep[:case["max_keep"]].numpy().astype(np.int32)
        print("nms %-28s valid %6d, kept %5d, max_keep %d" % (name, vi.numel(), keep.numel(), case["max_keep"]))
    # MultiScaleRoIAlign at 7 and 14
    P = DC.roi_pyramid()
    boxes, count = DC.roi_boxes()
    feats = {str(i): p for i, p in enumerate(P)}
    for size in (7, 14):
        pooler = MultiScaleRoIAlign(["0", "1", "2", "3"], size, 2)
        y = pooler(feats, [boxes[:count]], [DC.ROI_IMAGE_HW])
        lv = pooler.map_levels([boxes[:count]])
        assert pooler.scales == [0.25, 0.125, 0.0625, 0.03125], pooler.scales
        out["roi/%d/levels" % size] = lv.numpy().astype(np.int32)
        out["roi/%d/feats" % size] = y[:, ::8, ::3, ::3].numpy() if size == 14 else y[:, ::4, ::2, ::2].numpy()
    print("roi levels", np.bincount(out["roi/7/levels"], minlength=4))
    # box candidates
    for name, case in DC.box_candidate_cases().items():
        pred, props = case["pred"], case["props"]
        b = det_utils.BoxCoder((10.0, 10.0, 5.0, 5.0)).decode(pred[:, DC.NC:DC.NC * 5], [props])
        b = box_ops.clip_boxes_to_image(b, case["clip_hw"])[:, 1:].reshape(-1, 4)
        s = torch.softmax(pred[:, :DC.NC], -1)[:, 1:].reshape(-1)
        live = (torch.arange(pred.shape[0]) < case["count"]).repeat_interleave(DC.NC - 1)
        small = torch.zeros(b.shape[0], dtype=torch.bool)
        small[box_ops.remove_small_boxes(b, R.BOX_MIN)] = True
        valid = live & (s > R.BOX_SCORE) & small
        near = int(((s - R.BOX_SCORE).abs() < 1e-6).sum())
        assert near == 0, "%s: %d scores within 1e-6 of the threshold" % (name, near)
        out["box/%s/valid" % name] = valid.numpy()
        out["box/%s/boxes" % name] = b[::5].numpy()
        out["box/%s/scores" % name] = s[::5].numpy()
        print("box %-10s valid %d, most in one row %d" % (name, int(valid.sum()), int(valid.view(-1, DC.NC - 1).sum(1).max())))
    # paste
    for name, case in DC.paste_cases().items():
        n = case["count"]
        ob = resize_boxes(case["boxes"][:n], list(case["from_hw"]), list(case["to_hw"]))
        m = paste_masks_in_image(case["probs"][:n, None], ob, tuple(case["to_hw"]), padding=1)
        out["paste/%s/boxes" % name] = ob.numpy()
        out["paste/%s/nonzero" % name] = np.packbits(m.numpy() != 0)
        out["paste/%s/masks" % name] = m[:, :, ::5, ::5].numpy()
    # transform: normalise + resize (the padding to 32 is the GPU kernel's own zero fill)
    for name, img in DC.transform_cases().items():
        t = GeneralizedRCNNTransform(800, 1333, list(R.MEAN), list(R.STD)).eval()
        x, _ = t.resize(t.normalize((img + 1) / 2.0), None)
        out["transform/%s/hw" % name] = np.array(x.shape[-2:], np.int32)
        out["transform/%s/image" % name] = x[:, ::31, ::31].numpy()
    save_npz(OUT, out)
    print("wrote %s (%.1f KB)" % (OUT, os.path.getsize(OUT) / 1e3))


if __name__ == "__main__":
    main()
