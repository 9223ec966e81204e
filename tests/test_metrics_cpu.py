"""oracle/metrics_ref.py against the golden made from the reference's own PNetLin (tests/golden/make_metrics_golden.py),
and its SSIM / PSNR restatement against hand-worked cases."""
import os

import numpy as np
import pytest
import torch

import metrics_cases as MC
from oracle import metrics_ref as R

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz"))
C1, C2 = (0.01 * 2) ** 2, (0.03 * 2) ** 2


def test_inputs_and_weights_regenerate_bit_for_bit():
    convs, lins = MC.synthetic_alexnet(), MC.synthetic_lins()
    assert MC.sha256(*[t for wb in convs for t in wb], *lins) == GOLD["weights_sha"].item()
    for name in MC.CASES:
        assert MC.sha256(*MC.make_case(name)) == GOLD[name + "/sha"].item(), name


@pytest.mark.parametrize("name", sorted(MC.CASES))
def test_oracle_matches_golden(name):
    preds, gts = MC.make_case(name)
    np.testing.assert_allclose(R.ssim_scores(preds, gts), GOLD[name + "/ssim"], rtol=0, atol=1e-12)
    np.testing.assert_array_equal(R.psnr_scores(preds, gts), GOLD[name + "/psnr"])
    if name == "rand512":
        return                                                        # the 512 px LPIPS is checked on the GPU only
    convs, lins = MC.synthetic_alexnet(), MC.synthetic_lins()
    torch.set_grad_enabled(False)
    val, layers = R.lpips(torch.from_numpy(gts) * 2 - 1, torch.from_numpy(preds) * 2 - 1, convs, lins)
    np.testing.assert_allclose(val.numpy(), GOLD[name + "/lpips"], rtol=0, atol=1e-10)
    np.testing.assert_allclose(layers.numpy(), GOLD[name + "/lpips_layers"], rtol=0, atol=1e-10)


def test_oracle_calculate_score_weighs_chunks_like_the_reference():
    preds, gts = MC.make_case("batch33")
    convs, lins = MC.synthetic_alexnet(), MC.synthetic_lins()
    torch.set_grad_enabled(False)
    s = R.perceptual_calculate_score(preds, gts, convs, lins)
    assert abs(s - GOLD["batch33/calculate_score"].item()) < 1e-10
    per = GOLD["batch33/lpips"]
    assert abs(s - (per[:32].mean() + per[32:].mean()) / 2) < 1e-10
    assert abs(s - per.mean()) > 1e-6                                 # the single-frame chunk weighs 16x more


def test_golden_special_cases():
    assert np.all(GOLD["identical/ssim"] == 1.0) and np.all(np.isinf(GOLD["identical/psnr"]))
    assert np.all(GOLD["identical/lpips"] == 0.0)
    _, gts = MC.make_case("nonneg")
    assert (gts * 2 - 1).min() >= 0


def _frame(v, s=32):
    return np.full((3, s, s), v, dtype=np.float32)


def test_constant_offset_by_hand():
    """ref = 0.25, pred = 0.75 everywhere (in [-1,1]): every window has zero variance, S = A1 / B1."""
    gt, pred = _frame(0.625), _frame(0.875)
    a, b = 0.25, 0.75
    expect = (2 * a * b + C1) / (a * a + b * b + C1)
    assert abs(R.structural_similarity(R.preprocess(pred), R.preprocess(gt)) - expect) < 1e-12
    # min(ref) >= 0: data_range 1, mse 0.25
    assert abs(R.peak_signal_noise_ratio(R.preprocess(gt), R.preprocess(pred)) - 10 * np.log10(1 / 0.25)) < 1e-12
    # ref below 0 switches data_range to 2
    gt2, pred2 = _frame(0.375), _frame(0.625)
    assert abs(R.peak_signal_noise_ratio(R.preprocess(gt2), R.preprocess(pred2)) - 10 * np.log10(4 / 0.25)) < 1e-12


@pytest.mark.parametrize("pos,windows", [((16, 16), 49), ((0, 0), 1), ((1, 10), 14)])
def test_single_pixel_change_by_hand(pos, windows):
    """ref = 0 (in [-1,1]); pred differs by d at one pixel of channel 0.  Each 7x7 window holding it has ux = d/49,
    vx = d^2/49, uy = vy = vxy = 0, so S = C1 C2 / ((ux^2 + C1)(vx + C2)); every other window has S = 1.  Only windows
    centred 3 or more pixels from the border count: 49 for an inner pixel, 1 for the corner, 14 for (1, 10)."""
    s, d = 32, 0.5
    gt = _frame(0.5, s)
    pred = gt.copy()
    pred[0][pos] = 0.5 + d / 2
    ux, vx = d / 49, d * d / 49
    S = C1 * C2 / ((ux * ux + C1) * (vx + C2))
    n = (s - 6) ** 2
    expect = ((n - windows + windows * S) / n + 2.0) / 3
    assert abs(R.structural_similarity(R.preprocess(pred), R.preprocess(gt)) - expect) < 1e-12
    mse = d * d / (3 * s * s)
    assert abs(R.peak_signal_noise_ratio(R.preprocess(gt), R.preprocess(pred)) - 10 * np.log10(1 / mse)) < 1e-9
