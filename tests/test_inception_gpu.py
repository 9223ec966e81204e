"""The InceptionV3 kernels (csrc/inception.cu, the slice max-pool) and impersonator_b200.metrics' InceptionFeatures,
FIDMetric and InceptionScoreMetric against the golden of the reference's own InceptionV3 / fid_score_func /
is_score_func and against oracle/inception_ref.py in float64."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import inception_cases as IC
from impersonator_b200 import kernels as K, metrics as M
from oracle import inception_ref as R

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inception.npz"))


@pytest.fixture(scope="module")
def sd():
    return IC.golden_state_dict(GOLD)


@pytest.fixture(scope="module")
def net(cuda, sd):
    return M.InceptionFeatures(cuda, weights=sd)


@pytest.mark.parametrize("hw", [(256, 256), (512, 512), (299, 299), (184, 328), (7, 5)])
def test_input_matches_interpolate(cuda, hw):
    g = torch.Generator().manual_seed(hw[0])
    x = torch.rand((2, 3) + hw, generator=g)
    out = K.inception_input(x.to(cuda))
    ref = F.interpolate(x.to(cuda) * 2 - 1, size=(299, 299), mode='bilinear', align_corners=False)
    ref64 = F.interpolate((x * 2 - 1).double(), size=(299, 299), mode='bilinear', align_corners=False)
    err = (out - ref).abs().max().item()
    err64 = (out.cpu().double() - ref64).abs().max().item()
    print("%s: input vs F.interpolate %.1e (vs float64, whose source coordinates differ by float32 rounding: %.1e)"
          % (hw, err, err64))
    assert err < 1e-6 and err64 < 1e-4
    out = out.cpu()
    if hw == (299, 299):
        assert torch.equal(out, x * 2 - 1)


@pytest.mark.parametrize("box", [False, True])
def test_bn_act_segment_matches_float64(cuda, box):
    g = torch.Generator().manual_seed(5)
    raw = torch.rand((2, 9, 11, 200), generator=g) * 8 - 4
    scale, shift = torch.rand(48, generator=g) + 0.5, torch.rand(48, generator=g) - 0.5
    c0, off, pitch = 24, 16, 128
    y = torch.full((2, 9, 11, pitch), 7.0, device=cuda)
    hi = torch.full(y.shape, 7.0, dtype=torch.float16, device=cuda)
    lo = torch.full_like(hi, 7.0)
    K.bn_act_segment(raw.to(cuda), c0, 48, scale.to(cuda), shift.to(cuda), relu=True, box=box, c_out=64, y_f32=y,
                     y_hi=hi, y_lo=lo, off_y=off)
    r = raw[..., c0:c0 + 48].double()
    if box:
        r = F.avg_pool2d(r.permute(0, 3, 1, 2), 3, 1, 1).permute(0, 2, 3, 1)
    ref = F.relu(r * scale.double() + shift.double())
    y, hi, lo = y.cpu(), hi.cpu(), lo.cpu()
    err = (y[..., off:off + 48].double() - ref).abs().max().item() / ref.abs().max().item()
    print("box=%s: epilogue vs float64 %.1e relative" % (box, err))
    assert err < 1e-6
    v = y[..., off:off + 48]
    assert torch.equal(hi[..., off:off + 48], v.half()) and torch.equal(lo[..., off:off + 48], (v - v.half().float()).half())
    assert torch.all(y[..., off + 48:off + 64] == 0) and torch.all(hi[..., off + 48:off + 64] == 0)
    assert torch.all(y[..., :off] == 7) and torch.all(y[..., off + 64:] == 7) and torch.all(lo[..., off + 64:] == 7)


def test_maxpool_slice_exact(cuda):
    g = torch.Generator().manual_seed(6)
    x = (torch.rand((2, 35, 35, 320), generator=g) * 8 - 4).to(cuda)
    ref = F.max_pool2d(x[..., :288].permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1)
    hi = torch.full((2, 17, 17, 768), 3.0, dtype=torch.float16, device=cuda)
    lo = torch.full_like(hi, 3.0)
    y = torch.full((2, 17, 17, 768), 3.0, device=cuda)
    K.maxpool_nhwc_slice(x, 288, 3, 2, y_f32=y, y_hi=hi, y_lo=lo, off_y=480)
    assert torch.equal(y[..., 480:], ref)
    assert torch.equal(hi[..., 480:], ref.half()) and torch.equal(lo[..., 480:], (ref - ref.half().float()).half())
    assert torch.all(y[..., :480] == 3) and torch.all(hi[..., :480] == 3)


@pytest.mark.parametrize("name", sorted(IC.CASES))
def test_features_match_golden(cuda, net, name):
    f = net(torch.from_numpy(IC.make_case(name)).to(cuda)).cpu().double().numpy()
    g = GOLD[name + "/feats"]
    err = (np.abs(f - g).max(1) / np.abs(g).max(1)).max()
    print("%s: features vs reference %.1e of max|f| per frame" % (name, err))
    assert f.shape == g.shape and err < 1e-4


def test_stages_match_oracle(cuda, net, sd):
    frames = IC.make_case("rand256")
    taps = {}
    ref = R.features(frames, sd, device=cuda, taps=taps)
    f = net(torch.from_numpy(frames).to(cuda))
    st = net.stream(*frames.shape[:1], *frames.shape[2:])
    mine = dict(stem=st.stem, mixed_5d=st.mixed_5d[..., :288], mixed_6e=st.mixed_6e)
    for k, v in mine.items():
        r = taps[k].permute(0, 2, 3, 1)
        err = (v.double() - r).abs().max().item() / r.abs().max().item()
        print("%s vs float64 oracle: %.1e of max" % (k, err))
        assert err < (1e-5 if k == "stem" else 1e-4), k
    err = (f.double() - ref).abs().max().item() / ref.abs().max().item()
    print("mixed_7c (pooled) vs float64 oracle: %.1e of max" % err)
    assert err < 1e-4


def test_features_repeat_bit_for_bit(cuda, net):
    x = torch.from_numpy(IC.make_case("rand256")).to(cuda)
    assert torch.equal(net(x), net(x))


def test_metric_classes_and_calculate_score(cuda, sd):
    preds, gts = IC.make_batch33()
    fid = M.FIDMetric(cuda, weights=sd)
    s = fid.calculate_score(preds, gts)                                   # numpy in, chunks of 32 and 1
    ref = GOLD["batch33/fid"].item()
    print("batch33 FID %.6f, relative to the golden %.1e" % (s, abs(s - ref) / ref))
    assert isinstance(s, float) and abs(s - ref) < 1e-4 * ref
    ism = M.InceptionScoreMetric(cuda, weights=sd)
    m, sdv = ism.calculate_score(torch.from_numpy(preds).to(cuda))
    gm, gs = GOLD["batch33/is"]
    print("batch33 IS (%.8f, %.8f), golden (%.8f, %.8f)" % (m, sdv, gm, gs))
    assert abs(m - gm) < 1e-4 * gm and abs(sdv - gs) < 1e-4 * gm       # one chunk of one frame scores exactly 1
    f = fid.forward(preds[:3])
    p = ism.forward(preds[:3])
    assert isinstance(f, np.ndarray) and f.dtype == np.float32 and f.shape == (3, 2048)
    assert p.dtype == np.float32 and np.allclose(p.sum(1), 1, atol=1e-5)
    assert fid.quality() == 'lower score is better.' and ism.quality() == 'higher score is better'


@pytest.mark.parametrize("name", sorted(IC.FEATS))
def test_device_frechet_and_is_match_golden(cuda, name):
    a, b = (torch.from_numpy(t).to(cuda) for t in IC.make_feats(name))
    torch.cuda.synchronize()
    fid = M.FIDMetric.fid_score_func(a, b)
    ref, ref_eig = GOLD["feats/%s/fid" % name].item(), GOLD["feats/%s/fid_eig" % name].item()
    rel = abs(fid - ref) / abs(ref) if math.isfinite(ref) else float("nan")
    print("%s: device FID %.6f, relative to the reference %.1e, to the eig route %.1e"
          % (name, fid, rel, abs(fid - ref_eig) / abs(ref_eig)))
    assert abs(fid - ref_eig) < 1e-6 * abs(ref_eig)
    if math.isfinite(ref):
        assert rel < 1e-6
    score = M.InceptionScoreMetric.is_score_func(torch.softmax(a * IC.IS_GAIN, dim=1))
    ref_is = GOLD["feats/%s/is" % name].item()
    kl_rel = abs(math.log(score) - math.log(ref_is)) / math.log(ref_is)
    print("%s: mean KL (log IS) relative %.1e" % (name, kl_rel))
    assert kl_rel < 1e-6


def test_missing_weights_name_the_file(cuda, tmp_path, monkeypatch):
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    with pytest.raises(M.LwbError, match="inception_v3_google-0cc3c7bd.pth"):
        M.InceptionFeatures(cuda)
    with pytest.raises(M.LwbError, match="inception_v3_google-1a9a5a14.pth"):
        M.FIDMetric(cuda)
    with pytest.raises(M.LwbError, match="my_inception.pth"):
        M.load_inception_weights(str(tmp_path / "my_inception.pth"))
