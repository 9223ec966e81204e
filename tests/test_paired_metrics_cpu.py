"""The paired-metric contract cases (paired_metric_cases.py) on the CPU: the long-double SSIM / PSNR reference against
oracle/metrics_ref.py and the golden, the restatement of k_ssim_tiles + k_ssim_finish against the bars, and the
strength of those bars: every mutant of the restatement, and every wrong LPIPS variant, exceeds them at least 4x."""
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import metrics_cases as MC
import paired_metric_cases as P
from oracle import metrics_ref as R

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz"))
SMALL = [c for c in P.CASES if c.n <= 64]                          # the restatement holds a float64 copy of every tile
ORACLE_FRAMES = 64                                                 # frames of the big batch scored by the oracle


@pytest.fixture(scope="module")
def refs():
    """edge -> (pred, ref, reference SSIM, reference PSNR)."""
    out = {}
    for c in P.CASES:
        pred, ref = P.make(c)
        out[c.edge] = (pred, ref) + P.ssim_psnr_ref(pred, ref, c.from01)
    return out


def test_cases_are_the_required_edges():
    edges = [c.edge for c in P.CASES]
    assert len(set(edges)) == len(edges) and sorted(edges) == sorted(P.REQUIRED_EDGES)
    assert {1, 3, 5} <= {c.n for c in P.CASES} and max(c.n for c in P.CASES) > P.MAX_FRAMES_PER_LAUNCH
    partial = [c for c in P.CASES if c.h % P.TILE_H or c.w % P.TILE_W]
    assert {c.from01 for c in partial} == {0, 1}
    assert {c.w % P.TILE_W for c in P.CASES} > {0} and {c.h % P.TILE_H for c in P.CASES} > {0}
    c = P.by_edge("14x70_crop_in_second_column_tile")                # the crop ends 3 columns into the second tile
    assert P.TILE_W < c.w - P.CROP < 2 * P.TILE_W


@pytest.mark.parametrize("content", ["min_zero", "min_neg_ulp", "min_neg_zero"])
def test_range_cases_put_min_ref_in_the_last_partial_tile_of_channel_2(content, refs):
    """min(ref) is one pixel in the last partial tile of channel 2 of the last frame; the data range follows numpy's
    min(ref) >= 0 (so -0.0 gives 1)."""
    v = np.float32(P.RANGE_MIN[content])
    for c in P.CASES:
        if c.content != content:
            continue
        pred, ref, _, psnr = refs[c.edge]
        x, y = P.preprocess(pred, c.from01), P.preprocess(ref, c.from01)
        assert y[-1, 2, -1, -1] == v and np.signbit(y[-1, 2, -1, -1]) == np.signbit(v)
        rest = y.copy()
        rest[-1, 2, -1, -1] = 1
        assert rest.min() > 0 and c.h % P.TILE_H and c.w % P.TILE_W
        rng = 1.0 if v >= 0 else 2.0
        mse = np.mean((y[-1] - x[-1]) ** 2, dtype=np.float64)
        assert abs(psnr[-1] - 10 * np.log10(rng * rng / mse)) < 1e-12


@pytest.mark.parametrize("case", P.CASES, ids=[c.edge for c in P.CASES])
def test_reference_matches_the_oracle(case, refs):
    """The long-double reference against oracle/metrics_ref.py (skimage restated with uniform_filter)."""
    pred, ref, s, p = refs[case.edge]
    frames = None
    if case.n > ORACLE_FRAMES:
        frames = list(range(ORACLE_FRAMES // 2)) + list(range(case.n - ORACLE_FRAMES // 2, case.n))
    os_, op = P.oracle_scores(pred, ref, case.from01, frames)
    idx = slice(None) if frames is None else frames
    rs, rp = P.err_over_bar(os_, s[idx], 1e-12), P.err_over_bar(op, p[idx], 1e-10)
    print("%s: oracle - reference: SSIM %.2e, PSNR %.2e dB" % (case.edge, rs.max() * 1e-12, rp.max() * 1e-10))
    assert rs.max() <= 1 and rp.max() <= 1


def test_reference_matches_the_golden():
    for name in sorted(MC.CASES):
        preds, gts = MC.make_case(name)
        s, p = P.ssim_psnr_ref(preds, gts, 1)
        rs = P.err_over_bar(s, GOLD[name + "/ssim"], 1e-12)
        rp = P.err_over_bar(p, GOLD[name + "/psnr"], 1e-10)
        print("%s: reference - golden: SSIM %.2e, PSNR %.2e dB" % (name, rs.max() * 1e-12, rp.max() * 1e-10))
        assert rs.max() <= 1 and rp.max() <= 1, name


def test_reference_by_hand():
    """Frames of constants: every window has zero variance, so S = A1 / B1.  In frame 1, min(ref) = -0.0 at the last
    pixel gives data range 1, as numpy's -0.0 >= 0 does."""
    pred = np.full((2, 3, 9, 70), 0.75, np.float32)
    ref = np.full((2, 3, 9, 70), 0.25, np.float32)
    ref[1, 2, 8, 69] = -0.0
    c1 = (P.K1 * 2) ** 2
    s, p = P.ssim_psnr_ref(pred, ref, 0)
    assert abs(s[0] - (2 * 0.75 * 0.25 + c1) / (0.75 ** 2 + 0.25 ** 2 + c1)) < 1e-15
    assert abs(p[0] - 10 * np.log10(1 / 0.25)) < 1e-12
    mse = (0.25 * (3 * 9 * 70 - 1) + 0.75 ** 2) / (3 * 9 * 70)
    assert abs(p[1] - 10 * np.log10(1 / mse)) < 1e-12


def _worst(ssim_psnr, case, refs):
    _, _, s, p = refs[case.edge]
    return max(P.err_over_bar(ssim_psnr[0], s, P.SSIM_BAR).max(), P.err_over_bar(ssim_psnr[1], p, P.PSNR_BAR).max())


@pytest.mark.parametrize("case", SMALL, ids=[c.edge for c in SMALL])
def test_restatement_meets_every_case(case, refs):
    pred, ref = refs[case.edge][:2]
    r = _worst(P.restated(pred, ref, case.from01), case, refs)
    print("%s: restatement err / bar %.3g" % (case.edge, r))
    assert r <= 1.0


@pytest.mark.parametrize("mutant", P.MUTANTS)
def test_mutant_exceeds_the_bar(mutant, refs):
    ratios = {c.edge: _worst(P.restated(refs[c.edge][0], refs[c.edge][1], c.from01, mutant), c, refs) for c in SMALL}
    for edge, r in sorted(ratios.items(), key=lambda kv: -kv[1])[:5]:
        print("%s / %s: err / bar %.3g" % (mutant, edge, r))
    best = max(ratios.values())
    print("%s: largest err / bar %.3g" % (mutant, best))
    assert best >= 4.0, "mutant %s stays within 4x the bar on every case (largest %.3g)" % (mutant, best)


def test_f32_moments_passed_the_old_bar():
    """Float32 window sums and map stay within the former 1e-6 SSIM bar on the golden's noisy cases: only the 1e-12
    bar tells them from the float64 kernel there."""
    for name in ("rand256", "rand512", "nonneg", "batch33"):
        preds, gts = MC.make_case(name)
        s, _ = P.restated(preds, gts, 1, "f32_moments")
        d = np.abs(s - GOLD[name + "/ssim"]).max()
        print("%s: f32_moments - golden SSIM %.2e (%.3g x the new bar)" % (name, d, d / P.SSIM_BAR))
        assert 4 * P.SSIM_BAR < d < 1e-6


# ---- LPIPS ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def weights():
    return MC.synthetic_alexnet(), MC.synthetic_lins()


def _ceil_pools():
    """metrics_ref's torch.nn.functional with ceil-mode max pools."""
    ns = types.SimpleNamespace(**{k: getattr(F, k) for k in ("conv2d", "relu")})
    ns.max_pool2d = lambda x, k, s: F.max_pool2d(x, k, s, ceil_mode=True)
    return ns


VARIANTS = ["ceil_mode_pools", "lin_of_wrong_tap"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_lpips_variant_exceeds_the_bar(variant, weights, monkeypatch):
    """The LPIPS bar separates plausible wrong networks at the new sizes: ceil-mode pools, and tap 3's lin weights
    swapped with tap 4's (both 256 channels)."""
    convs, lins = weights
    lins_v = list(lins)
    if variant == "lin_of_wrong_tap":
        lins_v[3], lins_v[4] = lins[4], lins[3]
    worst = {}
    for c in P.LPIPS_CASES:
        pred, ref = P.make_lpips(c)
        val, layers = P.lpips_ref(pred, ref, c.from01, convs, lins)
        with monkeypatch.context() as m:
            if variant == "ceil_mode_pools":
                m.setattr(R, "F", _ceil_pools())
            v2, l2 = P.lpips_ref(pred, ref, c.from01, convs, lins_v)
        worst[c.edge] = max(np.abs(v2 - val).max(), np.abs(l2 - layers).max()) / P.LPIPS_BAR
        print("%s / %s: err / bar %.3g" % (variant, c.edge, worst[c.edge]))
    assert max(worst.values()) >= 4.0


def test_lpips_30x30_cannot_pool(weights):
    convs, lins = weights
    x = torch.zeros((1, 3) + P.LPIPS_REFUSED)
    with pytest.raises(RuntimeError):
        R.lpips(x, x, convs, lins)
    c = P.LPIPS_CASES[0]
    assert (c.h, c.w) == (31, 31)
    val, layers = P.lpips_ref(*P.make_lpips(c), c.from01, convs, lins)
    assert np.isfinite(val).all() and np.isfinite(layers).all()
