"""The paired-metric kernels (csrc/metrics.cu) against the float64 contract cases of paired_metric_cases.py:
k_ssim_tiles + k_ssim_finish against the long-double SSIM / PSNR reference at every tile, frame-size, content and
batch edge, and the LPIPS chain (k_lpips_input, the AlexNet features, k_lpips_layer) against oracle.metrics_ref.lpips
in float64 at the sizes where its features shrink to 1 x 1 .. 3 x 3."""
import numpy as np
import pytest
import torch

import metrics_cases as MC
import paired_metric_cases as P
from impersonator_b200 import kernels as K, metrics as M
from oracle import metrics_ref as R

pytestmark = pytest.mark.gpu


def _check(edge, got_s, got_p, want_s, want_p):
    rs, rp = P.err_over_bar(got_s, want_s, P.SSIM_BAR), P.err_over_bar(got_p, want_p, P.PSNR_BAR)
    print("%s: SSIM %.2e (err / bar %.3g), PSNR %.2e dB (err / bar %.3g)"
          % (edge, rs.max() * P.SSIM_BAR, rs.max(), rp.max() * P.PSNR_BAR, rp.max()))
    # NaN and +-inf match exactly (err_over_bar is inf where they do not)
    assert rs.max() <= 1.0 and rp.max() <= 1.0, edge


@pytest.mark.parametrize("case", P.CASES, ids=[c.edge for c in P.CASES])
def test_ssim_psnr_match_the_reference(cuda, case):
    pred, ref = P.make(case)
    want_s, want_p = P.ssim_psnr_ref(pred, ref, case.from01)
    p, r = torch.from_numpy(pred).to(cuda), torch.from_numpy(ref).to(cuda)
    s, q = K.ssim_psnr(p, r, from01=bool(case.from01))
    s, q = s.cpu().numpy(), q.cpu().numpy()
    _check(case.edge, s, q, want_s, want_p)
    s2, q2 = M.ssim_psnr(pred, ref, from01=bool(case.from01))          # numpy in: one copy to the device
    assert np.array_equal(s2.cpu().numpy(), s, equal_nan=True) and np.array_equal(q2.cpu().numpy(), q, equal_nan=True)
    if case.content == "identical":
        assert np.all(s == 1.0) and np.all(q == np.inf)


def test_nan_and_inf_stay_in_their_frames(cuda):
    """A NaN in frame 1's pred gives NaN SSIM and PSNR there, a +inf in frame 3's NaN SSIM and -inf PSNR; every other
    frame scores bit for bit as in the same batch without them."""
    case = P.by_edge("nan_inf_isolation")
    (pred, ref), (clean, _) = P.make(case), P.make(case, clean=True)
    s, q = (t.cpu().numpy() for t in K.ssim_psnr(torch.from_numpy(pred).to(cuda), torch.from_numpy(ref).to(cuda),
                                                 from01=True))
    s0, q0 = (t.cpu().numpy() for t in K.ssim_psnr(torch.from_numpy(clean).to(cuda), torch.from_numpy(ref).to(cuda),
                                                   from01=True))
    nan_i, inf_i = P.NAN_AT[0], P.INF_AT[0]
    assert np.isnan(s[nan_i]) and np.isnan(q[nan_i])
    assert np.isnan(s[inf_i]) and q[inf_i] == -np.inf
    others = [i for i in range(case.n) if i not in (nan_i, inf_i)]
    assert np.all(np.isfinite(s0)) and np.all(np.isfinite(q0))
    assert s[others].tobytes() == s0[others].tobytes() and q[others].tobytes() == q0[others].tobytes()


def test_metric_classes_score_more_frames_than_one_launch_holds(cuda):
    """21846 frames: past the 21845 that fit one k_ssim_tiles launch (3 planes per frame on grid.z)."""
    case = P.by_edge("batch_21846_frames")
    assert case.n > P.MAX_FRAMES_PER_LAUNCH and case.from01
    pred, ref = P.make(case)
    want_s, want_p = P.ssim_psnr_ref(pred, ref, 1)
    s = M.SSIMMetric().calculate_score(pred, ref)
    p = M.PSNRMetric().calculate_score(pred, ref)
    print("21846 frames: SSIM mean %.2e, PSNR mean %.2e dB" % (abs(s - want_s.mean()), abs(p - want_p.mean())))
    assert abs(s - want_s.mean()) <= P.SSIM_BAR and abs(p - want_p.mean()) <= P.PSNR_BAR
    # the frames of the second launch score as they do alone
    tail = slice(P.MAX_FRAMES_PER_LAUNCH - 2, None)
    s_all, p_all = (t.cpu().numpy() for t in M.ssim_psnr(pred, ref))
    s_tail, p_tail = (t.cpu().numpy() for t in M.ssim_psnr(pred[tail], ref[tail]))
    assert s_all[tail].tobytes() == s_tail.tobytes() and p_all[tail].tobytes() == p_tail.tobytes()


# ---- LPIPS ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def weights():
    return MC.synthetic_alexnet(), MC.synthetic_lins()


@pytest.fixture(scope="module")
def lp(cuda, weights):
    convs, lins = weights
    return M.LPIPS(cuda, weights=MC.alexnet_state_dict(convs), lin_weights=MC.lin_state_dict(lins))


@pytest.mark.parametrize("case", P.LPIPS_CASES, ids=[c.edge for c in P.LPIPS_CASES])
def test_lpips_matches_the_oracle(cuda, lp, weights, case):
    pred, ref = P.make_lpips(case)
    val, layers = P.lpips_ref(pred, ref, case.from01, *weights)
    score, lay = lp(torch.from_numpy(pred).to(cuda), torch.from_numpy(ref).to(cuda), from01=bool(case.from01))
    d = np.abs(score.cpu().double().numpy() - val).max()
    d_lay = np.abs(lay.cpu().double().numpy() - layers).max(axis=0)
    print("%s: LPIPS %.2e (err / bar %.3g), layers %s"
          % (case.edge, d, d / P.LPIPS_BAR, " ".join("%.1e" % v for v in d_lay)))
    assert d <= P.LPIPS_BAR and d_lay.max() <= P.LPIPS_BAR


def test_perceptual_calculate_score_at_an_odd_size(cuda, weights):
    """33 frames of 43 x 61: chunks of 32 and 1, the single-frame chunk weighing as much as the other."""
    case = next(c for c in P.LPIPS_CASES if c.n == 33)
    assert case.from01
    convs, lins = weights
    pred, ref = P.make_lpips(case)
    pm = M.PerceptualMetric(cuda, weights=MC.alexnet_state_dict(convs), lin_weights=MC.lin_state_dict(lins))
    got = float(pm.calculate_score(pred, ref))
    with torch.no_grad():
        want = R.perceptual_calculate_score(pred, ref, convs, lins, dtype=torch.float64)
    print("calculate_score, 33 frames of 43x61: %.2e" % abs(got - want))
    assert abs(got - want) <= P.LPIPS_BAR


def test_lpips_refuses_30x30(cuda, lp):
    x = torch.zeros((1, 3) + P.LPIPS_REFUSED, device=cuda)
    with pytest.raises(M.LwbError, match="too small"):
        lp(x, x)
