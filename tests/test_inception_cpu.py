"""oracle/inception_ref.py and the float64 torch score functions of impersonator_b200.metrics on CPU tensors, against
the golden made from the reference's own InceptionV3, fid_score_func and is_score_func
(tests/golden/make_inception_golden.py)."""
import math
import os

import numpy as np
import pytest
import torch

import inception_cases as IC
from impersonator_b200 import metrics as M
from oracle import inception_ref as R

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inception.npz"))


def test_inputs_and_weights_regenerate_bit_for_bit():
    assert IC.sha256(*[t for p in IC.synthetic_inception().values() for t in p]) == GOLD["weights_sha"].item()
    assert IC.sha256(IC.make_frames(*IC.CALIB)) == GOLD["calib_sha"].item()
    for name in IC.CASES:
        assert IC.sha256(IC.make_case(name)) == GOLD[name + "/sha"].item(), name
    assert IC.sha256(*IC.make_batch33()) == GOLD["batch33/sha"].item()
    for name in IC.FEATS:
        assert IC.sha256(*IC.make_feats(name)) == GOLD["feats/%s/sha" % name].item(), name


@pytest.mark.parametrize("name", sorted(IC.CASES))
def test_oracle_features_match_golden(name):
    f = R.features(IC.make_case(name), IC.golden_state_dict(GOLD), map_dtype=torch.float64).numpy()
    g = GOLD[name + "/feats"]
    err = np.abs(f - g).max() / np.abs(g).max()
    print("%s: oracle vs reference features %.1e of max|f|" % (name, err))
    assert err < 1e-10


def test_loader_folds_batchnorm_and_validates_shapes():
    sd = IC.golden_state_dict(GOLD)
    convs = M.load_inception_weights(sd)
    assert len(convs) == 94
    w, scale, shift = convs["Mixed_6c.branch7x7_2"]
    assert tuple(w.shape) == (160, 160, 1, 7)
    p = "Mixed_6c.branch7x7_2.bn."
    s64 = sd[p + "weight"].double() / torch.sqrt(sd[p + "running_var"].double() + 0.001)
    assert torch.equal(scale, s64.float())
    assert torch.equal(shift, (sd[p + "bias"].double() - sd[p + "running_mean"].double() * s64).float())
    bad = dict(sd)
    bad["Mixed_7c.branch3x3_2b.conv.weight"] = torch.zeros(384, 384, 1, 3)
    with pytest.raises(M.LwbError, match="Mixed_7c.branch3x3_2b.conv.weight"):
        M.load_inception_weights(bad)
    del bad["Mixed_5b.branch_pool.bn.running_var"]
    with pytest.raises(M.LwbError, match="Mixed_5b.branch_pool.bn.running_var"):
        M.load_inception_weights(bad)


@pytest.mark.parametrize("name", sorted(IC.FEATS))
def test_torch_frechet_and_is_on_cpu_match_golden(name):
    a, b = IC.make_feats(name)
    fid = M.FIDMetric.fid_score_func(torch.from_numpy(a), torch.from_numpy(b))
    ref, ref_eig = GOLD["feats/%s/fid" % name].item(), GOLD["feats/%s/fid_eig" % name].item()
    assert isinstance(fid, float)
    assert abs(fid - ref_eig) < 1e-9 * abs(ref_eig)
    if math.isfinite(ref):
        print("%s: FID %.6f, relative to the reference %.1e" % (name, fid, abs(fid - ref) / abs(ref)))
        assert abs(fid - ref) < 1e-6 * abs(ref)
    probs = torch.softmax(torch.from_numpy(a) * IC.IS_GAIN, dim=1)
    score = M.InceptionScoreMetric.is_score_func(probs)
    ref_is = GOLD["feats/%s/is" % name].item()
    assert abs(math.log(score) - math.log(ref_is)) < 1e-6 * math.log(ref_is)
    assert abs(M.InceptionScoreMetric.is_score_func(probs.numpy()) - score) < 1e-12 * score


@pytest.mark.parametrize("name", ["d64_n500", "d8_n50"])
def test_oracle_frechet_restatement_matches_golden(name):
    a, b = IC.make_feats(name)
    assert abs(R.fid(a, b) - GOLD["feats/%s/fid" % name].item()) < 1e-9 * GOLD["feats/%s/fid" % name].item()
    p = R.softmax64(a * IC.IS_GAIN)
    assert abs(R.inception_score(p) - GOLD["feats/%s/is" % name].item()) < 1e-12


def test_rank_deficient_and_degenerate_sets():
    # 33 frames in 2048 dimensions: rank-32 covariances; the reference's sqrtm of their product and the eigenvalue
    # route agree to 1e-5 here (on other rank-deficient sets the reference's imaginary-part check raises)
    ref, eig = GOLD["batch33/fid"].item(), GOLD["batch33/fid_eig"].item()
    assert abs(ref - eig) < 1e-5 * eig
    a, _ = IC.make_feats("d8_n50")
    t = torch.from_numpy(a)
    assert M.FIDMetric.fid_score_func(t, t) == pytest.approx(0.0, abs=1e-9)
    assert M.FIDMetric.fid_score_func(t[:0], t) == 0.0 and M.FIDMetric.fid_score_func([], []) == 0.0
    with pytest.raises(M.LwbError, match="at least 2 frames"):
        M.FIDMetric.fid_score_func(t[:1], t)
    mu, s = t.mean(0), torch.from_numpy(np.cov(a, rowvar=False))
    assert M.FIDMetric.calculate_frechet_distance(mu.numpy(), s.numpy(), mu, s) == pytest.approx(0.0, abs=1e-9)
