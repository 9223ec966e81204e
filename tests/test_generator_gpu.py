"""End-to-end GPU parity of the generator mirror (wgmma conv engine + fused LWB) against
  * the slices the REFERENCE modules produced (tests/golden/generator.npz), and
  * the full outputs of the functional restatement (oracle/generator_ref.py) on CPU.
Bar (BASELINE.json north_star): 1e-3 max-abs on fp32 pixels, met by the default fp16f8 mode and by fp16x3."""
import os

import numpy as np
import pytest
import torch

from impersonator_b200 import synthetic as S
from impersonator_b200.generator import ImpersonatorGenerator
from oracle import generator_ref as G

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-3


def sl(t):
    return t[:, :, 3::8, 5::8].cpu().numpy()


@pytest.fixture(scope="module")
def net(cuda):
    torch.set_grad_enabled(False)
    n = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    sd = S.fill_state_dict(n.state_dict(), seed=0)
    n.load_state_dict(sd)
    return n.to(cuda).eval(), sd


def test_inference_matches_reference_golden_and_oracle(cuda, net):
    """encode_src + inference (networks/generator.py:213-214, 277-301), B=2 targets, 1 source."""
    n, sd = net
    g = np.load(os.path.join(GOLD, "generator.npz"))
    inp = S.synthetic_generator_inputs(2, 256, seed=21)
    enc, res = n.encode_src(inp["src"].to(cuda))
    img, mask = n.inference(enc, res, inp["tsf"].to(cuda), inp["T"].to(cuda))
    torch.cuda.synchronize()
    d_img = np.abs(sl(img) - g["inf_tsf_img"]).max()
    d_mask = np.abs(sl(mask) - g["inf_tsf_mask"]).max()
    d_enc = np.abs(enc[3][:, ::16, ::4, ::4].cpu().numpy() - g["inf_enc3"]).max()
    d_res = np.abs(res[5][:, ::16, ::4, ::4].cpu().numpy() - g["inf_res5"]).max()
    print("vs reference golden: tsf_img %.3e tsf_mask %.3e enc3 %.3e res5 %.3e" % (d_img, d_mask, d_enc, d_res))
    assert d_img < TOL and d_mask < TOL and d_enc < TOL and d_res < 5 * TOL
    e_o, r_o = G.encode_src(inp["src"], sd)
    img_o, mask_o = G.inference(e_o, r_o, inp["tsf"], inp["T"], sd)
    f_img = (img.cpu() - img_o).abs().max().item()
    f_mask = (mask.cpu() - mask_o).abs().max().item()
    print("vs oracle full tensors: tsf_img %.3e tsf_mask %.3e" % (f_img, f_mask))
    assert f_img < TOL and f_mask < TOL
    bg = torch.rand(1, 3, 256, 256) * 2 - 1
    _, _, pred = n.inference(enc, res, inp["tsf"].to(cuda), inp["T"].to(cuda), bg=bg.to(cuda))
    ref_pred = mask_o * bg + (1 - mask_o) * img_o                          # models/imitator.py:331
    assert (pred.cpu() - ref_pred).abs().max().item() < TOL


def test_forward_matches_reference_golden(cuda, net):
    """Full ImpersonatorGenerator.forward (bg + src + tsf streams), BASELINE config 1."""
    n, sd = net
    g = np.load(os.path.join(GOLD, "generator.npz"))
    inp = S.synthetic_generator_inputs(1, 256, seed=11)
    outs = n(inp["bg"].to(cuda), inp["src"].to(cuda), inp["tsf"].to(cuda), inp["T"].to(cuda))
    torch.cuda.synchronize()
    for name, t in zip(("img_bg", "src_img", "src_mask", "tsf_img", "tsf_mask"), outs):
        d = np.abs(sl(t) - g["fwd_" + name]).max()
        print("forward %-9s vs reference golden: %.3e" % (name, d))
        assert d < TOL


def test_fast_mode_reports_its_error(cuda, net, monkeypatch):
    """Single-pass fp16 ("fast") mode: measured, not parity-gated (SURVEY.md 0.4)."""
    n, sd = net
    monkeypatch.setenv("LWB_PRECISION", "fp16")
    g = np.load(os.path.join(GOLD, "generator.npz"))
    inp = S.synthetic_generator_inputs(2, 256, seed=21)
    enc, res = n.encode_src(inp["src"].to(cuda))
    img, mask = n.inference(enc, res, inp["tsf"].to(cuda), inp["T"].to(cuda))
    d_img = np.abs(sl(img) - g["inf_tsf_img"]).max()
    d_mask = np.abs(sl(mask) - g["inf_tsf_mask"]).max()
    print("fast mode vs reference golden: tsf_img %.3e tsf_mask %.3e" % (d_img, d_mask))
    assert d_img < 5e-2 and d_mask < 5e-2


def test_swap_matches_oracle(cuda, net):
    """ImpersonatorGenerator.swap (two LWB warps per site, networks/generator.py:245-275)."""
    n, sd = net
    a = S.synthetic_generator_inputs(1, 256, seed=31)
    b = S.synthetic_generator_inputs(1, 256, seed=41)
    e12, r12 = n.encode_src(a["src"].to(cuda))
    e21, r21 = n.encode_src(b["src"].to(cuda))
    img, mask = n.swap(a["tsf"].to(cuda), e12, e21, r12, r21, a["T"].to(cuda), b["T"].to(cuda))
    eo12, ro12 = G.encode_src(a["src"], sd)
    eo21, ro21 = G.encode_src(b["src"], sd)
    img_o, mask_o = G.swap(a["tsf"], eo12, eo21, ro12, ro21, a["T"], b["T"], sd)
    d1, d2 = (img.cpu() - img_o).abs().max().item(), (mask.cpu() - mask_o).abs().max().item()
    print("swap vs oracle: %.3e %.3e" % (d1, d2))
    assert d1 < TOL and d2 < TOL
    g = np.load(os.path.join(GOLD, "generator.npz"))            # the reference modules' own swap() on the same inputs
    g1, g2 = np.abs(sl(img) - g["swap_img"]).max(), np.abs(sl(mask) - g["swap_mask"]).max()
    print("swap vs reference golden: %.3e %.3e" % (g1, g2))
    assert g1 < TOL and g2 < TOL


@pytest.mark.parametrize("mode", ["fp16f8", "fp16x3"])
def test_both_parity_modes_meet_the_bar(cuda, net, monkeypatch, mode):
    """fp16f8 (default): main product in fp16, both small products in e4m3 (2 instead of 3 MMA passes);
    fp16x3: all three products in fp16.  Same 1e-3 bar against the reference golden, on inference
    (config 2/3 path) and the full forward (config 1)."""
    n, sd = net
    monkeypatch.setenv("LWB_PRECISION", mode)
    g = np.load(os.path.join(GOLD, "generator.npz"))
    inp = S.synthetic_generator_inputs(2, 256, seed=21)
    enc, res = n.encode_src(inp["src"].to(cuda))
    img, mask = n.inference(enc, res, inp["tsf"].to(cuda), inp["T"].to(cuda))
    d = {"tsf_img": np.abs(sl(img) - g["inf_tsf_img"]).max(), "tsf_mask": np.abs(sl(mask) - g["inf_tsf_mask"]).max(),
         "enc3": np.abs(enc[3][:, ::16, ::4, ::4].cpu().numpy() - g["inf_enc3"]).max(),
         "res5": np.abs(res[5][:, ::16, ::4, ::4].cpu().numpy() - g["inf_res5"]).max()}
    print("%s vs reference golden (inference): %s" % (mode, d))
    assert d["tsf_img"] < TOL and d["tsf_mask"] < TOL and d["enc3"] < TOL and d["res5"] < 5 * TOL
    inp = S.synthetic_generator_inputs(1, 256, seed=11)
    outs = n(inp["bg"].to(cuda), inp["src"].to(cuda), inp["tsf"].to(cuda), inp["T"].to(cuda))
    for name, t in zip(("img_bg", "src_img", "src_mask", "tsf_img", "tsf_mask"), outs):
        dd = np.abs(sl(t) - g["fwd_" + name]).max()
        print("%s forward %-9s vs reference golden: %.3e" % (mode, name, dd))
        assert dd < TOL


def test_align_corners_opt_in_matches_installed_torch_golden(cuda, net, monkeypatch):
    """LWB_ALIGN_CORNERS=0: the flag-less F.grid_sample of the reference as torch >= 1.3 evaluates it (ac0_* goldens:
    the reference modules run unpatched under the installed torch)."""
    n, sd = net
    monkeypatch.setenv("LWB_ALIGN_CORNERS", "0")
    g = np.load(os.path.join(GOLD, "generator.npz"))
    inp = S.synthetic_generator_inputs(1, 256, seed=11)
    outs = n(inp["bg"].to(cuda), inp["src"].to(cuda), inp["tsf"].to(cuda), inp["T"].to(cuda))
    for name, t in zip(("img_bg", "src_img", "src_mask", "tsf_img", "tsf_mask"), outs):
        d = np.abs(sl(t) - g["ac0_fwd_" + name]).max()
        print("align_corners=0 forward %-9s vs reference golden: %.3e" % (name, d))
        assert d < TOL
    # and the two conventions really differ on the warped stream
    assert np.abs(g["fwd_tsf_img"] - g["ac0_fwd_tsf_img"]).max() > 1e-2


@pytest.mark.parametrize("tag,B,size,seed,step", [("b16_256", 16, 256, 61, 16), ("b8_512", 8, 512, 71, 32)])
def test_baseline_sizes_match_reference_golden(cuda, net, tag, B, size, seed, step):
    """BASELINE configs[2] (batch 16 @256) and configs[4] (batch 8 @512): encode_src + inference against slices and
    per-frame means of what the REFERENCE modules produced at those sizes (tests/golden/generator_big.npz)."""
    n, sd = net
    g = np.load(os.path.join(GOLD, "generator_big.npz"))
    inp = S.synthetic_generator_inputs(B, size, seed=seed)
    enc, res = n.encode_src(inp["src"].to(cuda))
    img, mask = n.inference(enc, res, inp["tsf"].to(cuda), inp["T"].to(cuda))
    torch.cuda.synchronize()
    d_img = np.abs(img[:, :, 3::step, 5::step].cpu().numpy() - g[tag + "_img"]).max(axis=(1, 2, 3))
    d_mask = np.abs(mask[:, :, 3::step, 5::step].cpu().numpy() - g[tag + "_mask"]).max(axis=(1, 2, 3))
    d_mean = np.abs(img.mean(dim=(1, 2, 3)).cpu().numpy() - g[tag + "_img_mean"])
    d_amean = np.abs(img.abs().mean(dim=(1, 2, 3)).cpu().numpy() - g[tag + "_img_absmean"])
    print("%s per-frame max-abs vs reference golden: img %s mask %s; means %.2e %.2e"
          % (tag, np.array2string(d_img, precision=1), np.array2string(d_mask, precision=1), d_mean.max(), d_amean.max()))
    assert d_img.shape[0] == B
    assert d_img.max() < TOL and d_mask.max() < TOL              # every one of the B frames
    assert d_mean.max() < 1e-4 and d_amean.max() < 1e-4
    assert not (n.range_status() & 3)


def test_tensor_core_heads_equal_cuda_core_heads(cuda, net, monkeypatch):
    """The 7x7 heads folded onto the tensor cores (7x1 filter, N = 7 columns x 4 channels) against the fp32 CUDA-core kernel."""
    n, sd = net
    inp = S.synthetic_generator_inputs(2, 256, seed=21)
    enc, res = n.encode_src(inp["src"].to(cuda))
    monkeypatch.setenv("LWB_TC_HEADS", "1")
    n._lwb_invalidate()
    img1, mask1 = n.inference(enc, res, inp["tsf"].to(cuda), inp["T"].to(cuda))
    img1, mask1 = img1.clone(), mask1.clone()
    monkeypatch.setenv("LWB_TC_HEADS", "0")
    n._lwb_invalidate()
    img0, mask0 = n.inference(enc, res, inp["tsf"].to(cuda), inp["T"].to(cuda))
    d = max((img1 - img0).abs().max().item(), (mask1 - mask0).abs().max().item())
    print("tensor-core heads vs CUDA-core heads: %.3e" % d)
    n._lwb_invalidate()
    assert d < 2e-4


def test_sub_batch_streams_match_single_stream(cuda, net, monkeypatch):
    """LWB_STREAMS=2: the batch runs as two sub-batches on side streams (their kernels overlap); same frames, same
    results up to the order of the fp64 InstanceNorm atomics."""
    n, sd = net
    inp = S.synthetic_generator_inputs(8, 256, seed=33)
    enc, res = n.encode_src(inp["src"].to(cuda))
    bg = (torch.rand(1, 3, 256, 256) * 2 - 1).to(cuda)
    tsf, T = inp["tsf"].to(cuda), inp["T"].to(cuda)
    monkeypatch.setenv("LWB_STREAMS", "1")
    c1, m1, p1 = [t.clone() for t in n.inference(enc, res, tsf, T, bg=bg)]
    monkeypatch.setenv("LWB_STREAMS", "2")
    hwc = torch.empty(8, 256, 256, 3, device=cuda)
    u8 = torch.empty(8, 256, 256, 3, dtype=torch.uint8, device=cuda)
    for _ in range(3):                                       # repeated: the side streams must be ordered against the caller's
        c2, m2, p2 = n.inference(enc, res, tsf, T, bg=bg, pred_hwc=hwc, pred_u8=u8)
    torch.cuda.synchronize()
    d = max((c1 - c2).abs().max().item(), (m1 - m2).abs().max().item(), (p1 - p2).abs().max().item())
    print("two sub-batch streams vs one: %.3e" % d)
    assert any(k[0].startswith("inference#") for k in n.tsf_model._lwb_streams), "the sub-batch streams were not used"
    assert d < 1e-5
    assert torch.equal(hwc, p2.permute(0, 2, 3, 1))
    assert not (n.range_status() & 3)


def test_captured_graph_survives_stream_cache_eviction(cuda, net):
    """A captured step replays into the buffers of the per-shape stream it was recorded with.  Nine other batch sizes push
    that shape out of the 8-entry stream cache; the graph must still own its buffers (graph.pin) and reproduce the eager
    result bit for bit."""
    from impersonator_b200.graph import CapturedStep
    n, _ = net
    size = 128
    inp = S.synthetic_generator_inputs(3, size, seed=31)
    enc, res = n.encode_src(inp["src"][:1].to(cuda))
    tsf, T = inp["tsf"].to(cuda), inp["T"].to(cuda)
    want_img, want_mask = [t.clone() for t in n.inference(enc, res, tsf, T)]

    step = CapturedStep(lambda tsf, T: n.inference(enc, res, tsf, T), dict(tsf=tsf, T=T))
    assert step.captured and step.pinned
    for B in (1, 2, 4, 5, 6, 7, 9, 10, 11):
        other = S.synthetic_generator_inputs(B, size, seed=40 + B)
        n.inference(enc, res, other["tsf"].to(cuda), other["T"].to(cuda))
    keys = [k for k in n.tsf_model._lwb_streams if k[1] == 3]
    assert not keys, "the B=3 stream should have been evicted: %r" % (keys,)
    junk = [torch.full((64, 1024, 1024), 7.0, device=cuda) for _ in range(4)]     # would land in freed buffers
    img, mask = step(tsf=tsf, T=T)
    torch.cuda.synchronize()
    assert torch.equal(img, want_img) and torch.equal(mask, want_mask)
    del junk


def test_captured_graph_keeps_the_workspaces_it_replays_into(cuda):
    """correspond and smpl_forward run on per-device cached workspaces, which a larger call replaces.  A step captured
    around both (as the Imitator's chunk graph is) must keep the buffers it replays into (graph.pin) when an eager B = 16
    call grows both caches; its replay then reproduces the eager result bit for bit and writes into no tensor allocated
    after the growth."""
    import glue_cases
    from impersonator_b200 import kernels as K
    from impersonator_b200.graph import CapturedStep
    from impersonator_b200.nmr import SMPLRenderer
    from oracle import nmr_ref
    size = 256
    v, f = S.uv_sphere()
    r = SMPLRenderer(image_size=size, faces=f.numpy(), map_fn=S.synthetic_tables()["map_fn"]).to(cuda)
    model = {k: t.to(cuda) for k, t in glue_cases.smpl_device_model(glue_cases.smpl_model(5, 6890)).items()}
    cam_s, verts_s = S.synthetic_frames(1, seed=60, base_verts=v)
    p2v = nmr_ref.src_p2verts(nmr_ref.project_to_faces(cam_s, verts_s, f)).contiguous().to(cuda)
    src = S.synthetic_source(size).to(cuda)

    def inputs(B, seed):
        cam, verts = S.synthetic_frames(B, seed=seed, base_verts=v)
        g = torch.Generator().manual_seed(seed)
        return dict(cam=cam.to(cuda), verts=verts.to(cuda), beta=torch.randn(B, 10, generator=g).to(cuda),
                    theta=(0.4 * torch.randn(B, 72, generator=g)).to(cuda))

    def step_fn(cam, verts, beta, theta):
        c = r.correspond(cam, verts, p2v, src)
        sv, sj, _, _, _ = K.smpl_forward(beta, theta, model)
        return c["fim"], c["wim"], c["T"], c["tsf_inputs"], sv, sj

    small = inputs(2, 61)
    idx = small["cam"].device.index
    kinds = ("raster", "smpl")
    for kind in kinds:                                   # start from empty caches: B = 2 sizes them, B = 16 grows them
        K._ws_cache.pop((idx, kind), None)
    want = [t.clone() for t in step_fn(**small)]
    step = CapturedStep(step_fn, small)
    assert step.captured
    ptrs = {kind: K._ws_cache[(idx, kind)].data_ptr() for kind in kinds}
    nbytes = {kind: K._ws_cache[(idx, kind)].numel() for kind in kinds}
    step_fn(**inputs(16, 62))
    torch.cuda.synchronize()
    pinned = {t.data_ptr() for t in step.pinned if torch.is_tensor(t)}
    for kind in kinds:
        assert K._ws_cache[(idx, kind)].data_ptr() != ptrs[kind], "the B = 16 call did not replace the %s workspace" % kind
        assert ptrs[kind] in pinned, "the captured step does not keep the %s workspace it replays into" % kind
    junk = [torch.full((nbytes[kind],), 7, dtype=torch.uint8, device=cuda) for kind in kinds for _ in range(4)]
    got = step(**small)
    torch.cuda.synchronize()
    for name, a, b in zip(("fim", "wim", "T", "tsf_inputs", "smpl verts", "smpl joints"), got, want):
        assert torch.equal(a, b), name
    assert all(bool((j == 7).all()) for j in junk), "the replay wrote into a tensor allocated after the capture"
