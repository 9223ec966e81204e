"""End-to-end GPU parity of the Imitator mirror (models/imitator.py:82-189) against the oracle:
personalize -> chunked inference over several target frames, host in / host out."""
import numpy as np
import pytest
import torch

from impersonator_b200 import synthetic as S
from impersonator_b200.generator import ImpersonatorGenerator
from impersonator_b200.imitator import Imitator, SyntheticBodyModel, morph
from impersonator_b200.nmr import SMPLRenderer
from oracle import generator_ref as G, nmr_ref

pytestmark = pytest.mark.gpu


class Opt(object):
    image_size, batch_size, bg_model, repeat_num, cond_nc = 256, 2, "ORIGINAL", 6, 3
    bg_ks, ft_ks, front_warp, only_vis = 13, 3, False, False


def ref_morph(mask, ks, mode='erode'):            # utils/util.py:73-89 verbatim (F.conv2d with a box kernel)
    import torch.nn.functional as F
    pad = ks // 2
    kernel = torch.ones(1, 1, ks, ks)
    if mode == 'erode':
        out = F.conv2d(F.pad(mask, [pad] * 4, value=1.0), kernel)
        return (out == ks * ks).float()
    out = F.conv2d(F.pad(mask, [pad] * 4, value=0.0), kernel)
    return (out >= 1).float()


def test_imitator_inference_matches_oracle(cuda):
    torch.set_grad_enabled(False)
    size = 256
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    net = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    sd = S.fill_state_dict(net.state_dict(), seed=0)
    net.load_state_dict(sd)
    render = SMPLRenderer(image_size=size, faces=f.numpy(), map_fn=tabs["map_fn"])
    body = SyntheticBodyModel(v)
    im = Imitator(Opt(), generator=net, hmr=body, render=render, device=cuda)
    src_img = S.synthetic_source(size)
    src_theta = np.zeros(85, np.float32)
    src_theta[0], src_theta[3], src_theta[4] = 0.95, 0.3, 0.1
    im.personalize("", src_smpl=src_theta, src_img=src_img)
    g = torch.Generator().manual_seed(5)
    tgt = np.zeros((5, 85), np.float32)
    tgt[:, 0] = 0.8 + 0.3 * torch.rand(5, generator=g).numpy()
    tgt[:, 1:3] = (torch.rand(5, 2, generator=g).numpy() * 2 - 1) * 0.1
    tgt[:, 3] = (torch.rand(5, generator=g).numpy() * 2 - 1) * 3.0
    tgt[:, 4] = (torch.rand(5, generator=g).numpy() * 2 - 1) * 0.3
    outs = im.inference_by_smpls(list(tgt), cam_strategy="smooth")          # chunks of 2, 2, 1
    assert len(outs) == 5 and outs[0].shape == (size, size, 3) and outs[0].dtype == np.float32

    # ---- oracle: the reference's personalize + per-frame loop (models/imitator.py:82-189), on CPU
    sth = torch.from_numpy(src_theta)[None]
    sinfo = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in body.get_details(sth.to(cuda)).items()}
    f2v, sfim, _ = nmr_ref.render_fim_wim(sinfo["cam"], sinfo["verts"], f, size)
    cond = nmr_ref.encode_fim(sfim, tabs["map_fn"])
    p2v = nmr_ref.src_p2verts(f2v)
    bg_mask = ref_morph(cond[:, -1:], 13, 'erode')
    bg = G.resnet_generator(torch.cat([src_img * bg_mask, bg_mask], dim=1), sd, 'bg_model')
    ft_mask = 1 - ref_morph(cond[:, -1:], 3, 'erode')
    feats = G.encode_src(torch.cat([src_img * ft_mask, cond], dim=1), sd)
    assert torch.equal(morph(cond[:, -1:], 13), bg_mask)
    first_cam = torch.from_numpy(tgt[0:1, 0:3])
    worst = 0.0
    for t in range(5):
        th = torch.from_numpy(tgt[t:t + 1])
        cam = sinfo["cam"].clone()
        cam[:, 1:] += th[:, 1:3] - first_cam[:, 1:]                          # swap_smpl 'smooth' (:224-227)
        tsf = body.get_details(torch.cat([cam, th[:, 3:75], sinfo["shape"]], dim=1).to(cuda))   # same device as the product path
        c = nmr_ref.correspond(tsf["cam"].cpu(), tsf["verts"].cpu(), f, tabs["map_fn"], p2v, src_img, size)
        pred, _, _ = G.imitator_forward(bg, feats, c["tsf_inputs"], c["T"], sd)
        d = np.abs(outs[t] - pred[0].permute(1, 2, 0).numpy()).max()
        worst = max(worst, d)
    print("Imitator.inference_by_smpls vs oracle loop: max-abs %.3e over 5 frames" % worst)
    assert worst < 1e-3
    assert im.tsf_info["T"].shape[0] == 1                                    # tsf_info describes the last frame


def test_imitator_batch16_every_frame_matches_oracle(cuda):
    """The headline configuration (BASELINE configs[2]): batch_size = 16, ONE chunk of 16 frames through
    Imitator.inference_by_smpls, every frame compared with the oracle's per-frame loop."""
    torch.set_grad_enabled(False)
    size, nf = 256, 16
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    net = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    sd = S.fill_state_dict(net.state_dict(), seed=0)
    net.load_state_dict(sd)
    render = SMPLRenderer(image_size=size, faces=f.numpy(), map_fn=tabs["map_fn"])
    body = SyntheticBodyModel(v)
    opt = Opt()
    opt.batch_size = 16
    im = Imitator(opt, generator=net, hmr=body, render=render, device=cuda)
    src_img = S.synthetic_source(size)
    src_theta = np.zeros(85, np.float32)
    src_theta[0], src_theta[3], src_theta[4] = 0.95, -0.4, 0.05
    im.personalize("", src_smpl=src_theta, src_img=src_img)
    g = torch.Generator().manual_seed(16)
    tgt = np.zeros((nf, 85), np.float32)
    tgt[:, 0] = 0.8 + 0.3 * torch.rand(nf, generator=g).numpy()
    tgt[:, 1:3] = (torch.rand(nf, 2, generator=g).numpy() * 2 - 1) * 0.1
    tgt[:, 3] = (torch.rand(nf, generator=g).numpy() * 2 - 1) * 3.0
    tgt[:, 4] = (torch.rand(nf, generator=g).numpy() * 2 - 1) * 0.3
    outs = im.inference_by_smpls(list(tgt), cam_strategy="smooth")
    assert len(outs) == nf

    sth = torch.from_numpy(src_theta)[None]
    sinfo = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in body.get_details(sth.to(cuda)).items()}
    f2v, sfim, _ = nmr_ref.render_fim_wim(sinfo["cam"], sinfo["verts"], f, size)
    cond = nmr_ref.encode_fim(sfim, tabs["map_fn"])
    p2v = nmr_ref.src_p2verts(f2v)
    bg_mask = ref_morph(cond[:, -1:], 13, 'erode')
    bg = G.resnet_generator(torch.cat([src_img * bg_mask, bg_mask], dim=1), sd, 'bg_model')
    ft_mask = 1 - ref_morph(cond[:, -1:], 3, 'erode')
    feats = G.encode_src(torch.cat([src_img * ft_mask, cond], dim=1), sd)
    first_cam = torch.from_numpy(tgt[0:1, 0:3])
    per_frame = []
    for t in range(nf):
        th = torch.from_numpy(tgt[t:t + 1])
        cam = sinfo["cam"].clone()
        cam[:, 1:] += th[:, 1:3] - first_cam[:, 1:]
        # the synthetic body model runs where the product ran it (cos / sin differ by an ulp between CPU and GPU, and a 1e-7
        # vertex shift can flip a silhouette pixel of the bit-exact rasterizer)
        tsf = body.get_details(torch.cat([cam, th[:, 3:75], sinfo["shape"]], dim=1).to(cuda))
        c = nmr_ref.correspond(tsf["cam"].cpu(), tsf["verts"].cpu(), f, tabs["map_fn"], p2v, src_img, size)
        pred, _, _ = G.imitator_forward(bg, feats, c["tsf_inputs"], c["T"], sd)
        per_frame.append(float(np.abs(outs[t] - pred[0].permute(1, 2, 0).numpy()).max()))
    print("Imitator batch 16 vs oracle loop, per-frame max-abs:", ["%.1e" % d for d in per_frame])
    assert max(per_frame) < 1e-3


def test_imitator_from_smpl_vectors_through_lbs_kernels(cuda):
    """85-float SMPL vectors in, frames out, with the SMPL LBS kernels as the body model (HumanModelRecovery.get_details,
    networks/hmr.py:302-330).  LBS parity itself is tests/test_smpl_gpu.py; here the oracle loop consumes the vertices the
    kernels produced, so that 1e-7 vertex differences cannot flip silhouette pixels of the bit-exact rasterizer."""
    from impersonator_b200.hmr import HumanModelRecovery
    from oracle import smpl_ref
    torch.set_grad_enabled(False)
    size = 256
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    net = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    sd = S.fill_state_dict(net.state_dict(), seed=0)
    net.load_state_dict(sd)
    render = SMPLRenderer(image_size=size, faces=f.numpy(), map_fn=tabs["map_fn"])
    dd = S.synthetic_smpl_model(seed=3)
    body = HumanModelRecovery(smpl_model=dd).to(cuda)
    opt = Opt()
    opt.batch_size = 3
    im = Imitator(opt, generator=net, hmr=body, render=render, device=cuda)
    src_img = S.synthetic_source(size)
    src_theta = S.synthetic_smpl_params(1, seed=5)
    im.personalize("", src_smpl=src_theta[0].numpy(), src_img=src_img)
    tgt = S.synthetic_smpl_params(4, seed=77)
    outs = im.inference_by_smpls(list(tgt.numpy()), cam_strategy="smooth")          # chunks of 3, 1
    assert len(outs) == 4
    assert im.tsf_info["j2d"].shape == (1, 19, 2) and im.tsf_info["verts"].shape == (1, 6890, 3)

    m = smpl_ref.model_tensors(dd)
    sinfo = smpl_ref.get_details(m, src_theta)
    assert (im.src_info["verts"].cpu() - sinfo["verts"]).abs().max() < 1e-5
    s_verts = im.src_info["verts"].cpu()
    f2v, sfim, _ = nmr_ref.render_fim_wim(sinfo["cam"], s_verts, f, size)
    cond = nmr_ref.encode_fim(sfim, tabs["map_fn"])
    p2v = nmr_ref.src_p2verts(f2v)
    bg_mask = ref_morph(cond[:, -1:], 13, 'erode')
    bg = G.resnet_generator(torch.cat([src_img * bg_mask, bg_mask], dim=1), sd, 'bg_model')
    ft_mask = 1 - ref_morph(cond[:, -1:], 3, 'erode')
    feats = G.encode_src(torch.cat([src_img * ft_mask, cond], dim=1), sd)
    first_cam = tgt[0:1, 0:3]
    worst = 0.0
    for t in range(4):
        th = tgt[t:t + 1]
        cam = sinfo["cam"].clone()
        cam[:, 1:] += th[:, 1:3] - first_cam[:, 1:]
        tsf_theta = torch.cat([cam, th[:, 3:75], sinfo["shape"]], dim=1)
        ref_verts = smpl_ref.get_details(m, tsf_theta)["verts"]
        gpu_verts = body.get_details(tsf_theta.to(cuda))["verts"].cpu()
        assert (gpu_verts - ref_verts).abs().max() < 1e-5
        c = nmr_ref.correspond(cam, gpu_verts, f, tabs["map_fn"], p2v, src_img, size)
        pred, _, _ = G.imitator_forward(bg, feats, c["tsf_inputs"], c["T"], sd)
        worst = max(worst, np.abs(outs[t] - pred[0].permute(1, 2, 0).numpy()).max())
    print("Imitator (SMPL LBS kernels) vs oracle loop: max-abs %.3e over 4 frames" % worst)
    assert worst < 1e-3


def _np_u8_bgr(frames_hwc):
    """utils/cv_utils.py:23-36 with normalize=True, minus the imwrite: RGB->BGR, ((img+1)/2.0*255).astype(uint8)."""
    img = frames_hwc[..., ::-1]
    return ((img + 1) / 2.0 * 255).astype(np.uint8)


def test_output_path_layouts(cuda):
    """SURVEY 8f rank 2: HWC float frames and BGR uint8 frames straight from the head kernel / lwb_frames_out."""
    from impersonator_b200 import kernels as K
    torch.set_grad_enabled(False)
    g = torch.Generator().manual_seed(3)
    frames = (torch.rand(3, 3, 64, 48, generator=g) * 2 - 1).to(cuda)
    frames[0, :, 0, 0] = torch.tensor([-1.0, 1.0, 0.0])
    hwc, u8 = K.frames_out(frames, want_hwc=True, want_u8=True)
    ref = frames.permute(0, 2, 3, 1).cpu().numpy()
    assert np.array_equal(hwc.cpu().numpy(), ref)
    assert np.array_equal(u8.cpu().numpy(), _np_u8_bgr(ref))
    raw = torch.randn(2, 32, 32, 4, generator=g).to(cuda)
    bg = (torch.rand(1, 3, 32, 32, generator=g) * 2 - 1).to(cuda)
    p_hwc = torch.empty(2, 32, 32, 3, device=cuda)
    p_u8 = torch.empty(2, 32, 32, 3, dtype=torch.uint8, device=cuda)
    color, mask, pred = K.heads_composite(raw, bg, pred_hwc=p_hwc, pred_u8=p_u8)
    assert torch.equal(p_hwc, pred.permute(0, 2, 3, 1))
    assert np.array_equal(p_u8.cpu().numpy(), _np_u8_bgr(p_hwc.cpu().numpy()))


def test_imitator_uint8_and_saved_frames(cuda, tmp_path):
    torch.set_grad_enabled(False)
    size = 256
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    net = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    net.load_state_dict(S.fill_state_dict(net.state_dict(), seed=0))
    render = SMPLRenderer(image_size=size, faces=f.numpy(), map_fn=tabs["map_fn"], has_front=True,
                          front_map_fn=tabs["front_map_fn"], back_map_fn=tabs["back_map_fn"])
    for front in (False, True):
        opt = Opt()
        opt.front_warp = front
        im = Imitator(opt, generator=net, hmr=SyntheticBodyModel(v), render=render, device=cuda)
        src_theta = np.zeros(85, np.float32)
        src_theta[0] = 0.95
        im.personalize("", src_smpl=src_theta, src_img=S.synthetic_source(size))
        tgt = np.zeros((3, 85), np.float32)
        tgt[:, 0], tgt[:, 3] = 0.9, np.array([0.2, 1.0, -2.0])
        assert im.inference_by_smpls([]) == [] and im.inference([], tgt_smpls=[]) == []      # empty sequence (the reference returns [])
        floats = im.inference_by_smpls(list(tgt))
        u8 = im.inference_by_smpls(list(tgt), as_uint8=True)
        assert u8[0].dtype == np.uint8 and u8[0].shape == (size, size, 3)
        for a, b in zip(floats, u8):
            assert np.array_equal(_np_u8_bgr(a), b)
        try:
            import cv2
        except ImportError:
            continue
        out = im.inference_by_smpls(list(tgt), output_dir=str(tmp_path))
        assert np.array_equal(out[1], floats[1])
        saved = cv2.imread(str(tmp_path / ("pred_%.8d.jpg" % 1)))
        assert saved is not None and saved.shape == (size, size, 3)
        expect = cv2.imdecode(cv2.imencode('.jpg', u8[1])[1], -1)                       # the same encoder, in memory
        assert np.array_equal(saved, expect)


def test_imitator_graph_replay_matches_eager(cuda, monkeypatch):
    """LWB_GRAPH: full chunks are replayed from a captured CUDA graph (SMPL LBS + raster + generator + composite); same frames
    as the eager launch sequence, sequence after sequence (first_cam / source buffers are read at fixed addresses), and a new
    source invalidates the graphs."""
    from impersonator_b200.hmr import HumanModelRecovery
    torch.set_grad_enabled(False)
    size = 256
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    net = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    net.load_state_dict(S.fill_state_dict(net.state_dict(), seed=0))
    render = SMPLRenderer(image_size=size, faces=f.numpy(), map_fn=tabs["map_fn"])
    body = HumanModelRecovery(smpl_model=S.synthetic_smpl_model(seed=3)).to(cuda)
    opt = Opt()
    opt.batch_size = 4
    im = Imitator(opt, generator=net, hmr=body, render=render, device=cuda)
    tgt_a, tgt_b = S.synthetic_smpl_params(10, seed=31), S.synthetic_smpl_params(8, seed=32)
    results = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("LWB_GRAPH", mode)
        im.personalize("", src_smpl=S.synthetic_smpl_params(1, seed=5)[0].numpy(), src_img=S.synthetic_source(size))
        a = im.inference_by_smpls(list(tgt_a.numpy()))                       # chunks 4, 4, 2 (the partial one runs eagerly)
        b = im.inference_by_smpls(list(tgt_b.numpy()), as_uint8=True)        # another first_cam, another layout
        im.personalize("", src_smpl=S.synthetic_smpl_params(1, seed=6)[0].numpy(), src_img=S.synthetic_source(size, seed=7))
        c = im.inference_by_smpls(list(tgt_b.numpy()))
        results[mode] = (a, b, c, im.tsf_info["T"].clone())
        if mode == "1":
            assert any(g.captured for g in im._graphs.values()), "the chunk graph was not captured"
    for x, y in zip(results["0"][0] + results["0"][2], results["1"][0] + results["1"][2]):
        assert np.abs(x - y).max() < 1e-5
    for x, y in zip(results["0"][1], results["1"][1]):
        assert np.abs(x.astype(np.int32) - y.astype(np.int32)).max() <= 1
    assert torch.equal(results["0"][3], results["1"][3])


def test_imitator_range_bits_redo_the_sequence_in_fp16x3_once(cuda, tmp_path, monkeypatch):
    """Operand-range bits from a pass: the generator is pinned to fp16x3 and the sequence is computed once more (the
    frames and files are that pass's, and its own bits are not checked again); LWB_AUTO_PRECISION=0 only warns, and
    RANGE_FP16 raises.  The bits are forced through a stand-in for the generator's range flag."""
    import warnings
    from impersonator_b200._lib import LwbError
    from impersonator_b200.binding import RANGE_FP16, RANGE_HEADS
    torch.set_grad_enabled(False)
    monkeypatch.delenv("LWB_PRECISION", raising=False)
    monkeypatch.delenv("LWB_AUTO_PRECISION", raising=False)
    size = 256
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    net = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    net.load_state_dict(S.fill_state_dict(net.state_dict(), seed=0))
    im = Imitator(Opt(), generator=net, hmr=SyntheticBodyModel(v),
                  render=SMPLRenderer(image_size=size, faces=f.numpy(), map_fn=tabs["map_fn"]), device=cuda)
    src_theta = np.zeros(85, np.float32)
    src_theta[0] = 0.95
    im.personalize("", src_smpl=src_theta, src_img=S.synthetic_source(size))
    tgt = np.zeros((3, 85), np.float32)
    tgt[:, 0], tgt[:, 3] = 0.9, np.array([0.2, 1.0, -2.0])
    flag = torch.full((1,), RANGE_HEADS, dtype=torch.int32, device=cuda)
    monkeypatch.setattr(im.generator.tsf_model, "range_flag_tensor", lambda: flag)

    def run(**kw):
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            outs = im.inference_by_smpls(list(tgt), **kw)
        return outs, [str(w.message) for w in rec if "lwb_b200" in str(w.message)]

    monkeypatch.setenv("LWB_AUTO_PRECISION", "0")
    outs, said = run()
    assert len(outs) == 3 and len(said) == 1 and "precision mode kept" in said[0]
    assert getattr(net, "_lwb_precision", None) is None
    monkeypatch.delenv("LWB_AUTO_PRECISION")
    outs, said = run(output_dir=str(tmp_path))
    assert len(outs) == 3 and len(said) == 1 and "switching this generator to LWB_PRECISION=fp16x3" in said[0]
    assert getattr(net, "_lwb_precision", None) == "fp16x3"
    flag.zero_()
    clean, said = run()
    assert said == [] and len(clean) == 3
    for a, b in zip(outs, clean):
        assert np.abs(a - b).max() < 1e-5
    assert sorted(p.name for p in tmp_path.iterdir()) == ["pred_%.8d.jpg" % t for t in range(3)]
    flag.fill_(RANGE_FP16)
    net.set_precision(None)
    with pytest.raises(LwbError, match="fp16 range"):
        run()
