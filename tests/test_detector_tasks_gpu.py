"""``--has_detector`` through the tasks: ``Imitator``, ``Viewer`` and ``Swapper`` built from synthetic asset files with the
flag set and synthetic Mask R-CNN weights in a temporary torch hub cache (where ``pretrained=True`` leaves them).
``personalize`` must take its background mask from the detector (models/imitator.py:116-122): the body mask equals the
oracle's (oracle/maskrcnn_ref.py on the same source image) except at pixels whose probability is within 1e-3 of the
threshold and their dilation footprint, and ``src_info['bg']`` is within 1e-3 of the background net run on that mask.
Then each task runs to its end."""
import numpy as np
import pytest
import torch

from impersonator_b200 import detectors as D, synthetic as S
from oracle import maskrcnn_ref as R

pytestmark = pytest.mark.gpu
SEED = 21


@pytest.fixture(scope="module")
def weights():
    return S.synthetic_maskrcnn_state(SEED)


def _check_background(task, weights):
    img = task.src_info['img']
    _, omask, det, _ = R.inference(img[0].cpu(), D.remap_v1(weights), ks=task._opt.bg_ks)
    pid = R.person_id(det["labels"], det["boxes"])
    near = (det["masks"][pid, 0] - 0.5).abs() < 1e-3
    excl = R.dilate(near.float()[None, None], task._opt.bg_ks)[0, 0] > 0
    _, gmask = task.detector.inference(img[0])
    gmask = gmask.cpu()
    assert int(((gmask != omask)[0, 0] & ~excl).sum()) == 0
    body = torch.where(excl, gmask[0, 0], omask[0, 0])[None, None].to(img.device)
    bg_mask = 1 - body
    bg_inputs = torch.cat([img * bg_mask, bg_mask], dim=1)
    want = task._original_bg(bg_inputs, task.bgnet(bg_inputs))
    assert (task.src_info['bg'] - want).abs().max().item() < 1e-3


@pytest.mark.parametrize("task_name", ["imitator", "viewer", "swapper"])
def test_tasks_with_has_detector(cuda, tmp_path, monkeypatch, weights, task_name):
    from test_run_imitator_gpu import reference_defaults
    torch.set_grad_enabled(False)
    hub = tmp_path / "hub"
    (hub / "checkpoints").mkdir(parents=True)
    torch.save(weights, str(hub / "checkpoints" / D.WEIGHTS_FILE))
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(hub))
    A = S.write_synthetic_assets(str(tmp_path))
    monkeypatch.chdir(tmp_path)
    opt = reference_defaults(src_path=A["src"], tgt_path=A["target_files"][0], load_path=A["load_path"], has_detector=True,
                             swap_part='body', view_params='R=0,90,0/t=0,0,0')
    if task_name == "imitator":
        from impersonator_b200.imitator import Imitator
        task = Imitator(opt)
        task.personalize(opt.src_path)
        assert isinstance(task.detector, D.PersonMaskRCNNDetector) and task.detector.ks == opt.bg_ks
        _check_background(task, weights)
        outs = task.inference([opt.tgt_path], tgt_smpls=None, cam_strategy='smooth', output_dir='', visualizer=None,
                              verbose=False)
        assert len(outs) == 1 and np.isfinite(outs[0]).all()
    elif task_name == "viewer":
        from impersonator_b200.viewer import Viewer
        task = Viewer(opt=opt)
        task.personalize(opt.src_path, visualizer=None)
        _check_background(task, weights)
        pred = task.view(np.array([0, np.pi / 2, 0], np.float32), np.zeros(3, np.float32), visualizer=None, name="0")
        assert pred.shape == (1, 3, 256, 256) and torch.isfinite(pred).all()
    else:
        from impersonator_b200.swapper import Swapper
        task = Swapper(opt=opt)
        task.swap_setup(opt.src_path, opt.tgt_path)
        _check_background(task, weights)
        preds = task.swap(src_info=task.src_info, tgt_info=task.tsf_info, target_part=opt.swap_part, visualizer=None)
        assert preds.shape == (1, 3, 256, 256) and torch.isfinite(preds).all()
