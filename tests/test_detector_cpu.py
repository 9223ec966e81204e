"""CPU checks of the Mask R-CNN person detector: the mirror's state_dict layout, the oracle against the golden made
from the reference's utils/detectors.py on torchvision (tests/golden/maskrcnn.npz), weight loading without downloads,
and the reference's person-selection quirks."""
import hashlib
import os

import numpy as np
import pytest
import torch

from impersonator_b200 import detectors as D, synthetic as S
from impersonator_b200._lib import LwbError
from oracle import maskrcnn_ref as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "maskrcnn.npz")


def source_image(golden, size):
    """The golden's source image: regenerated from its seed and checked against the digest the golden pins."""
    img = S.synthetic_source(size)[0]
    assert hashlib.sha256(np.ascontiguousarray(img.numpy()).tobytes()).hexdigest() == str(golden["s%d_img_sha256" % size])
    return img


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def weights(golden):
    return S.synthetic_maskrcnn_state(int(golden["seed"]))


def test_keys_and_shapes_match_both_layouts(golden, weights):
    m = D.MaskRCNN()
    assert sorted(m.state_dict()) == list(golden["keys_current"])
    assert sorted(weights) == list(golden["keys"])
    assert [str(tuple(weights[k].shape)) for k in sorted(weights)] == list(golden["shapes"])
    assert sum(v.numel() for v in weights.values()) == 44507633
    m.load_state_dict(weights)                                       # published (version-1) names
    m.load_state_dict(D.remap_v1(weights))                           # current names
    assert D.to_v1(D.remap_v1(weights)).keys() == weights.keys()


def test_oracle_reproduces_golden(golden, weights):
    torch.set_grad_enabled(False)
    img = source_image(golden, 256)
    box, mask, det, st = R.inference(img, D.remap_v1(weights), ks=13)
    assert np.abs(np.concatenate([p[0, :2, ::4, ::4].reshape(-1).numpy() for p in st["P"]]) - golden["s256_P_slices"]).max() < 1e-5
    lv = st["rpn"]["levels"]
    assert np.array_equal(np.concatenate([l["top"].numpy() for l in lv]), golden["s256_rpn_top"])
    assert np.abs(np.concatenate([l["logits"][:512].numpy() for l in lv]) - golden["s256_rpn_logits_head"]).max() < 1e-5
    assert np.abs(np.concatenate([l["deltas"][:128].numpy() for l in lv]) - golden["s256_rpn_deltas_head"]).max() < 1e-5
    assert np.abs(np.concatenate([l["proposals"][:128].numpy() for l in lv]) - golden["s256_rpn_proposals_head"]).max() < 1e-4
    assert np.abs(st["proposals"].numpy() - golden["s256_proposals"]).max() < 1e-4
    assert np.abs(st["class_logits"][:128].numpy() - golden["s256_class_logits_head"]).max() < 1e-5
    assert np.abs(st["box_regression"][:16].numpy() - golden["s256_box_regression_head"]).max() < 1e-5
    assert np.abs(st["mask_probs"][:8].numpy() - golden["s256_mask_probs_head"]).max() < 1e-5
    assert np.array_equal(det["labels"].numpy(), golden["s256_det_labels"].astype(np.int64))
    assert np.abs(det["boxes"].numpy() - golden["s256_det_boxes"]).max() < 1e-4
    assert np.abs(box.numpy() - golden["s256_box"]).max() < 1e-4
    assert np.array_equal(np.packbits(mask.numpy().astype(bool)), golden["s256_mask_bits"])


def test_golden_margins_clear_the_stage_bars(golden):
    for size in (256, 512):
        score, iou, area, _ = golden["s%d_margins" % size]
        assert min(score, iou, area) > 10 * 2e-4


def test_missing_weights_raise_without_download(tmp_path, monkeypatch):
    def no_download(*a, **k):
        raise AssertionError("the detector must never download")
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", no_download)
    monkeypatch.setattr(torch.hub, "download_url_to_file", no_download)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    with pytest.raises(LwbError, match=D.WEIGHTS_FILE):
        D.PersonMaskRCNNDetector(to_gpu=False)
    with pytest.raises(LwbError, match="nowhere.pth"):
        D.PersonMaskRCNNDetector(to_gpu=False, weights=str(tmp_path / "nowhere.pth"))


def test_weights_from_hub_cache_and_path(tmp_path, monkeypatch, weights):
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    os.makedirs(tmp_path / "checkpoints")
    torch.save(weights, str(tmp_path / "checkpoints" / D.WEIGHTS_FILE))
    det = D.PersonMaskRCNNDetector(ks=13, to_gpu=False)
    key = "roi_heads.box_predictor.cls_score.bias"
    assert torch.equal(det.model.state_dict()[key], weights[key])
    with pytest.raises(LwbError, match="CUDA"):
        det.inference(torch.zeros(3, 32, 32))


@pytest.mark.parametrize("labels,boxes,want", [
    ([1, 1, 3], [[0, 0, 10, 10], [0, 0, 20, 10], [0, 0, 50, 50]], 1),          # largest person
    ([1, 3, 1], [[0, 0, 10, 20], [0, 0, 50, 50], [0, 0, 20, 10]], 0),          # equal areas: the first wins
    ([2, 3, 4], [[0, 0, 10, 20], [0, 0, 50, 50], [0, 0, 20, 10]], -1),         # no person: -1 (the last detection)
])
def test_person_selection_quirks(labels, boxes, want):
    det = D.PersonMaskRCNNDetector.__new__(D.PersonMaskRCNNDetector)
    labels, boxes = torch.tensor(labels), torch.tensor(boxes, dtype=torch.float32)
    assert det.get_bbox_max_ids(labels, boxes) == want
    assert R.person_id(labels, boxes) == want
