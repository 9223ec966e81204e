"""The paired-metric kernels (csrc/metrics.cu, the 11x11 s4 direct stem, the floor-mode NHWC pool) and
impersonator_b200.metrics against the golden of the reference's PNetLin and oracle/metrics_ref.py."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import metrics_cases as MC
from impersonator_b200 import kernels as K, metrics as M
from oracle import metrics_ref as R

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz"))


@pytest.fixture(scope="module")
def lp(cuda):
    convs, lins = MC.synthetic_alexnet(), MC.synthetic_lins()
    return M.LPIPS(cuda, weights=MC.alexnet_state_dict(convs), lin_weights=MC.lin_state_dict(lins))


@pytest.mark.parametrize("name", sorted(MC.CASES))
def test_ssim_psnr_lpips_match_golden(cuda, lp, name):
    preds, gts = MC.make_case(name)
    p, g = torch.from_numpy(preds).to(cuda), torch.from_numpy(gts).to(cuda)
    ssim, psnr = M.ssim_psnr(p, g)
    ssim, psnr = ssim.cpu().numpy(), psnr.cpu().numpy()
    d_ssim = np.abs(ssim - GOLD[name + "/ssim"]).max()
    gp = GOLD[name + "/psnr"]
    assert np.array_equal(np.isinf(psnr), np.isinf(gp))
    fin = ~np.isinf(gp)
    d_psnr = np.abs(psnr[fin] - gp[fin]).max() if fin.any() else 0.0
    score, layers = lp(p, g)
    d_layers = np.abs(layers.cpu().numpy() - GOLD[name + "/lpips_layers"]).max(axis=0)
    d_lpips = np.abs(score.cpu().numpy() - GOLD[name + "/lpips"]).max()
    print("%s: SSIM %.2e, PSNR %.2e dB, LPIPS %.2e (layers %s)" % (name, d_ssim, d_psnr, d_lpips,
                                                                  " ".join("%.1e" % v for v in d_layers)))
    assert d_ssim < 1e-6 and d_psnr < 1e-4 and d_lpips < 1e-4 and d_layers.max() < 1e-4
    if name == "identical":
        assert np.all(ssim == 1.0) and np.all(np.isinf(psnr)) and np.all(score.cpu().numpy() == 0.0)


def test_scores_repeat_bit_for_bit(cuda, lp):
    preds, gts = MC.make_case("rand256")
    p, g = torch.from_numpy(preds).to(cuda), torch.from_numpy(gts).to(cuda)
    a, b = M.ssim_psnr(p, g), M.ssim_psnr(p, g)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(lp(p, g)[1], lp(p, g)[1])


def test_metric_classes_and_calculate_score(cuda, lp):
    preds, gts = MC.make_case("batch33")
    pm = M.PerceptualMetric(cuda, weights=MC.alexnet_state_dict(MC.synthetic_alexnet()),
                            lin_weights=MC.lin_state_dict(MC.synthetic_lins()))
    s = float(pm.calculate_score(preds, gts))                            # numpy in, chunks of 32 and 1
    assert abs(s - GOLD["batch33/calculate_score"].item()) < 1e-4
    assert abs(float(pm.calculate_score(torch.from_numpy(preds).to(cuda), torch.from_numpy(gts).to(cuda))) - s) < 1e-7
    assert abs(M.SSIMMetric().calculate_score(preds, gts) - GOLD["batch33/ssim"].mean()) < 1e-6
    assert abs(M.PSNRMetric().calculate_score(preds, gts) - GOLD["batch33/psnr"].mean()) < 1e-4
    assert abs(M.SSIMMetric().forward(preds[3], gts[3]) - GOLD["batch33/ssim"][3]) < 1e-6
    assert M.SSIMMetric().quality() == M.PSNRMetric().quality() == 'higher score is better'
    assert pm.quality() == 'lower score is better.'


def test_missing_weights_name_the_file(cuda, tmp_path):
    with pytest.raises(M.LwbError, match="alexnet-owt-7be5be79.pth"):
        M.load_alexnet_weights(str(tmp_path / "alexnet-owt-7be5be79.pth"))
    with pytest.raises(M.LwbError, match="alex.pth"):
        M.load_lin_weights(str(tmp_path / "alex.pth"))


def test_stem_11x11_s4_matches_conv2d(cuda):
    g = torch.Generator().manual_seed(3)
    x = torch.rand((2, 3, 131, 97), generator=g) * 4 - 2
    w, b = MC.synthetic_alexnet()[0]
    out = K.conv2d_direct_relu_nhwc(x.to(cuda), w.to(cuda), b.to(cuda), stride=4, pad=2)
    ref = F.relu(F.conv2d(x.double(), w.double(), b.double(), stride=4, padding=2)).permute(0, 2, 3, 1)
    err = (out.cpu().double() - ref).abs().max().item()
    print("11x11 s4 stem vs float64 conv2d: %.2e" % err)
    assert out.shape == ref.shape and err < 2e-5


def test_floor_pool_nhwc_exact(cuda):
    g = torch.Generator().manual_seed(4)
    for (h, w, c) in ((63, 63, 64), (31, 30, 192), (8, 7, 16)):
        x = (torch.rand((3, h, w, c), generator=g) * 8 - 4).to(cuda)
        ref = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1).contiguous()
        y = K.maxpool_nhwc(x, 3, 2)
        hi = torch.empty(ref.shape, dtype=torch.float16, device=cuda)
        lo = torch.empty_like(hi)
        K.maxpool_nhwc(x, 3, 2, y_hi=hi, y_lo=lo)
        assert torch.equal(y, ref)
        assert torch.equal(hi, ref.half()) and torch.equal(lo, (ref - ref.half().float()).half())


def test_imitator_score_against(cuda, lp):
    from impersonator_b200 import synthetic as S
    from impersonator_b200.generator import ImpersonatorGenerator
    from impersonator_b200.imitator import Imitator, SyntheticBodyModel
    from impersonator_b200.nmr import SMPLRenderer

    class Opt(object):
        image_size, batch_size, bg_model, repeat_num, cond_nc = 256, 2, "ORIGINAL", 6, 3
        bg_ks, ft_ks, front_warp, only_vis = 13, 3, False, False

    torch.set_grad_enabled(False)
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    net = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    net.load_state_dict(S.fill_state_dict(net.state_dict(), seed=0))
    im = Imitator(Opt(), generator=net, hmr=SyntheticBodyModel(v),
                  render=SMPLRenderer(image_size=256, faces=f.numpy(), map_fn=tabs["map_fn"]), device=cuda)
    src_theta = np.zeros(85, np.float32)
    src_theta[0], src_theta[3] = 0.95, 0.3
    im.personalize("", src_smpl=src_theta, src_img=S.synthetic_source(256))
    tgt = np.zeros((3, 85), np.float32)
    tgt[:, 0] = (0.8, 0.9, 1.0)
    tgt[:, 3] = (0.1, -0.4, 0.7)
    _, gts = MC.make_case("rand256")
    gt = torch.from_numpy(gts * 2 - 1)
    outs, scores = im.inference([""] * 3, tgt_smpls=list(tgt), score_against=gt, lpips=lp)     # chunks of 2, 1
    frames = torch.from_numpy(np.stack(outs)).permute(0, 3, 1, 2).contiguous().to(cuda)
    after = M.score_frames(frames, gt.to(cuda), lpips=lp)
    for k in ("ssim", "psnr"):
        assert np.array_equal(scores[k], after[k].cpu().numpy()), k
    assert np.abs(scores["lpips"] - after["lpips"].cpu().double().numpy()).max() < 1e-6
    assert set(scores) == {"ssim", "psnr", "lpips"} and scores["ssim"].shape == (3,)
