"""CPU checks of the detector's post-processing contract: oracle/maskrcnn_ref.py reproduces torchvision's own CPU ops on
every constructed case of tests/detector_cases.py (pinned in tests/golden/detector_cases.npz), and the ``lwb_det_*``
launchers reject bad arguments with LWB_E_INVALID and a message before any CUDA call.

Discrete outputs (top-k order, keep lists, levels, valid flags, the pasted region) must match exactly; float outputs
within 1e-6 of max|torchvision|."""
import ctypes
import os

import numpy as np
import pytest
import torch

import detector_cases as DC
from impersonator_b200 import _lib
from oracle import maskrcnn_ref as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "detector_cases.npz")


@pytest.fixture(scope="module")
def golden():
    torch.set_grad_enabled(False)
    return np.load(GOLD)


def close(got, want, rel=1e-6):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    assert np.abs(got - want).max(initial=0.0) <= rel * max(np.abs(want).max(initial=0.0), 1e-30)


def test_rpn_cases(golden):
    for name, case in DC.rpn_cases().items():
        for l, o in enumerate(DC.oracle_rpn(case)):
            p = "rpn/%s/%d/" % (name, l)
            assert np.array_equal(o["top"].numpy(), golden[p + "top"]), p
            assert np.array_equal(o["valid"].numpy(), golden[p + "valid"]), p
            close(o["boxes"][::7], golden[p + "boxes"])


def test_rpn_signed_zero_tie_is_by_index():
    """The k boundary falls inside 800 anchors at +-0: the stable sort takes them in index order, ignoring the sign."""
    case = DC.rpn_cases()["signed_zero_tie"]
    lg = (case["heads"][0][..., :3] + case["bias"][:3]).reshape(-1)
    top = DC.oracle_rpn(case)[0]["top"]
    zeros = torch.where(lg == 0)[0]
    chosen = top[lg[top] == 0]
    assert torch.equal(chosen, zeros[:chosen.numel()])
    assert bool((torch.signbit(lg[chosen])).any()) and bool((~torch.signbit(lg[chosen])).any())


def test_nms_cases(golden):
    for name, case in DC.nms_cases().items():
        assert np.array_equal(DC.oracle_nms(case).numpy(), golden["nms/%s/keep" % name]), name


def test_nms_thresholds_round_down():
    """The kernel compares the fp32 IoU with float(thresh), torchvision with the double thresh: the two agree exactly
    when float(thresh) <= thresh, which holds for both thresholds the detector uses."""
    for t in (R.RPN_NMS, R.BOX_NMS):
        assert float(np.float32(t)) <= t


def test_roi_align_cases(golden):
    P = DC.roi_pyramid()
    boxes, count = DC.roi_boxes()
    for size in (7, 14):
        y, lv = DC.oracle_roi_align(P, boxes, count, size)
        assert np.array_equal(lv.numpy(), golden["roi/%d/levels" % size].astype(np.int64))
        y = y[:count].permute(0, 3, 1, 2)
        close(y[:, ::8, ::3, ::3] if size == 14 else y[:, ::4, ::2, ::2], golden["roi/%d/feats" % size])
    # the sweep crosses every level boundary
    assert set(lv[:200].tolist()) == {0, 1, 2, 3}


def test_box_candidate_cases(golden):
    for name, case in DC.box_candidate_cases().items():
        b, s, g, v = DC.oracle_box_candidates(case)
        assert np.array_equal(v.numpy(), golden["box/%s/valid" % name]), name
        close(b[::5], golden["box/%s/boxes" % name])
        close(s[::5], golden["box/%s/scores" % name])
        # at most 19 classes of a row clear 0.05 (20 x 0.05 would be the whole softmax mass): m_max = 20 R is safe
        per_row = v.view(-1, DC.NC - 1).sum(1)
        assert int(per_row.max()) <= 19
    assert int(DC.oracle_box_candidates(DC.box_candidate_cases()["mixed"])[3].view(-1, DC.NC - 1).sum(1).max()) == 19


def test_paste_cases(golden):
    for name, case in DC.paste_cases().items():
        m, b = DC.oracle_paste(case)
        n = case["count"]
        assert np.array_equal(b[:n].numpy(), golden["paste/%s/boxes" % name]), name
        assert np.array_equal(np.packbits(m[:n].numpy() != 0), golden["paste/%s/nonzero" % name]), name
        close(m[:n, :, ::5, ::5], golden["paste/%s/masks" % name])


def test_transform_cases(golden):
    for name, img in DC.transform_cases().items():
        x, hw = R.transform((img + 1) / 2.0)
        assert list(hw) == golden["transform/%s/hw" % name].tolist()
        assert DC.detector_sizes(*img.shape[1:])[:2] == tuple(hw)
        close(x[0, :, :hw[0], :hw[1]][:, ::31, ::31], golden["transform/%s/image" % name])


# ---- launcher argument checks (no GPU) -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    return _lib.lib()


D = ctypes.c_void_p(1024)                # never dereferenced: every call below fails its argument check first


def _rejected(L, rc, text):
    assert rc == -1, rc
    assert text.encode() in L.lwb_last_error(), L.lwb_last_error()


def test_det_rpn_argument_checks(L):
    def rpn(levels=1, k=1000, heads=D):
        return L.lwb_det_rpn(levels, heads, D, D, D, D, D, D, D, k, 100.0, 100.0, 1e-3, 4.0, None, D, D, D, D, None)
    _rejected(L, rpn(k=1025), "k <= 1024")
    _rejected(L, rpn(k=0), "k <= 1024")
    _rejected(L, rpn(levels=6), "1..5 levels")
    _rejected(L, rpn(heads=None), "null pointer")


def test_det_nms_argument_checks(L):
    def nms(n=100, m_max=100, max_keep=10, ws=ctypes.c_void_p(4096), count=D):
        return L.lwb_det_nms(D, D, None, None, n, m_max, 0.5, max_keep, ws, D, None, None, None, count, None)
    _rejected(L, nms(ws=ctypes.c_void_p(4096 + 64)), "256-byte aligned")
    _rejected(L, nms(count=None), "null pointer")
    _rejected(L, nms(n=0), "bad sizes")
    _rejected(L, nms(max_keep=0), "bad sizes")
    _rejected(L, nms(m_max=64 * 6145), "too many boxes")
    # count | 3 x 129 ints | 129 boxes | 129 x 3 mask words, each section rounded up to 256 bytes
    assert L.lwb_det_nms_workspace_bytes(0, 129) == 256 + 3 * 768 + 2304 + 3328


def test_det_count_is_required(L):
    """The post-processing launchers read the number of live rows from a device count: a NULL count is refused."""
    _rejected(L, L.lwb_det_box_candidates(D, 464, 91, D, None, 10, 100.0, 100.0, 0.05, 0.01, 4.0, D, D, D, D, None), "null pointer")
    _rejected(L, L.lwb_det_mask_probs(D, 96, D, D, None, 10, 784, None, D, None), "null pointer")
    _rejected(L, L.lwb_det_paste_masks(D, 28, D, None, 10, 1.0, 1.0, 64, 64, D, D, None), "null pointer")
    _rejected(L, L.lwb_det_person_mask(D, D, None, 1, D, 64, 64, 0.5, 3, D, D, D, None), "null pointer")


def test_det_bad_sizes(L):
    _rejected(L, L.lwb_det_box_candidates(D, 400, 91, D, D, 10, 100.0, 100.0, 0.05, 0.01, 4.0, D, D, D, D, None), "bad sizes")
    _rejected(L, L.lwb_det_box_candidates(D, 464, 91, D, D, 0, 100.0, 100.0, 0.05, 0.01, 4.0, D, D, D, D, None), "bad sizes")
    _rejected(L, L.lwb_det_roi_align(D, D, D, 8, D, None, 0, 7, 2, None, D, None, None, None), "bad sizes")
    _rejected(L, L.lwb_det_mask_probs(D, 96, D, D, D, 0, 784, None, D, None), "bad sizes")
    _rejected(L, L.lwb_det_paste_masks(D, 0, D, D, 10, 1.0, 1.0, 64, 64, D, D, None), "bad sizes")
    _rejected(L, L.lwb_det_transform(D, 300, 300, 800, 800, 790, 800, D, None), "bad sizes")
    _rejected(L, L.lwb_det_stem_pool(D, 1, 64, 1, 9, D, D, D, D, None), "bad sizes")
    _rejected(L, L.lwb_det_bias_act(D, 8, None, None, None, 0, 1, 4, 4, 0, 1, 4, 4, 16, D, None, None, None), "bad sizes")
    _rejected(L, L.lwb_det_bias_act(D, 8, None, None, None, 0, 2, 5, 5, 0, 1, 4, 4, 8, D, None, None, None), "outside the input")
    _rejected(L, L.lwb_det_bias_act(D, 8, None, None, D, 1, 1, 5, 5, 0, 1, 5, 5, 8, D, None, None, None), "even grid")
    _rejected(L, L.lwb_det_d2s_bias_relu(D, D, 1, 0, 4, 8, D, None, None, None), "bad sizes")


@pytest.mark.parametrize("ks", [2, 4, 12])
def test_det_person_mask_rejects_even_ks(L, ks):
    """The reference's morph pads ks // 2 on every side: an even ks makes an (h+1) x (w+1) mask that its callers
    cannot combine with the h x w image.  The launcher refuses even ks instead of returning a shifted h x w mask."""
    _rejected(L, L.lwb_det_person_mask(D, D, D, 1, D, 64, 64, 0.5, ks, D, D, D, None), "ks must be 0 or odd")
    m = R.dilate(torch.zeros(1, 1, 8, 8), ks)
    assert m.shape[-2:] == (9, 9)
