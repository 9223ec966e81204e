"""Each ``K.det_*`` kernel of the Mask R-CNN detector on the constructed cases of tests/detector_cases.py, against the
torch-fp32 oracle (oracle/maskrcnn_ref.py, pinned to torchvision by tests/golden/detector_cases.npz), plus end-to-end
runs with zero detections, no person, and a stream reused across images.

Bars: discrete outputs (top-k order, keep lists, counts, levels, valid flags, the person pick and mask) exact; fp32
outputs built from __f*_rn operations (NMS boxes and scores, RoIAlign, bias_act, mask logits, the resized boxes) exact,
and their fp16 hi / lo operands the exact split of that value; outputs through expf (sigmoid, softmax, decode) within
a few ulps.  The input transform measures exact too; the stem pool and the paste, whose multiply-adds follow neither
torch's rounding nor ATen's operation order bit for bit, carry the bound measured on an H100."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import detector_cases as DC
from conv_emulation import fp16_pair
from impersonator_b200 import detectors as D, kernels as K, synthetic as S
from impersonator_b200._lib import LwbError
from oracle import maskrcnn_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def no_grad():
    torch.set_grad_enabled(False)


def i32(n, dev):
    return torch.tensor([n], dtype=torch.int32, device=dev)


def ulps(got, want):
    """Largest distance in units of want's last place."""
    got, want = got.detach().cpu().double(), want.detach().double()
    sp = torch.from_numpy(np.spacing(np.abs(want.float().numpy())).astype(np.float64))
    return float(((got - want).abs() / sp).max()) if want.numel() else 0.0


def box_ulps(got, want, scale):
    """Box corners: distance in ulps of the coordinate scale each corner was computed at (centre +- half size)."""
    sp = torch.from_numpy(np.spacing(np.abs(scale.float().numpy())).astype(np.float64))
    return float(((got.detach().cpu().double() - want.double()).abs() / sp[:, None]).max()) if want.numel() else 0.0


def assert_operands(hi, lo, v, what):
    wh, wl = fp16_pair(v)
    assert torch.equal(hi.cpu().view(torch.int16), wh.view(torch.int16)), what + " hi"
    assert torch.equal(lo.cpu().view(torch.int16), wl.view(torch.int16)), what + " lo"


# ---- RPN -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(DC.rpn_cases()))
def test_rpn(cuda, name):
    case = DC.rpn_cases()[name]
    want = DC.oracle_rpn(case)
    n = sum(o["top"].numel() for o in want)
    out = dict(boxes=torch.zeros((n, 4), device=cuda), scores=torch.zeros(n, device=cuda),
               groups=torch.zeros(n, dtype=torch.int32, device=cuda), valid=torch.zeros(n, dtype=torch.int32, device=cuda),
               top=torch.zeros(n, dtype=torch.int32, device=cuda))
    assert K.det_rpn([h.to(cuda) for h in case["heads"]], case["strides"], case["cells"], case["bias"].to(cuda), case["k"],
                     case["clip_hw"], case["min_size"], D.XFORM_CLIP, out) == n
    o = 0
    worst = dict(scores=0.0, boxes=0.0)
    for l, w in enumerate(want):
        k = w["top"].numel()
        sl = slice(o, o + k)
        assert torch.equal(out["top"][sl].cpu().long(), w["top"]), "level %d top-k" % l
        assert torch.equal(out["valid"][sl].cpu().bool(), w["valid"]), "level %d valid" % l
        assert bool((out["groups"][sl] == l).all())
        raw = R.decode(w["deltas"], w["anchors"], (1.0, 1.0, 1.0, 1.0))[:, 0]
        ctr = torch.stack([(raw[:, 0] + raw[:, 2]) / 2, (raw[:, 1] + raw[:, 3]) / 2], 1).abs()
        scale = torch.maximum(raw.abs().amax(1), ctr.amax(1))
        worst["boxes"] = max(worst["boxes"], box_ulps(out["boxes"][sl], w["boxes"], scale))
        worst["scores"] = max(worst["scores"], ulps(out["scores"][sl], w["scores"]))
        o += k
    print("rpn %s: sigmoid %.1f ulps, boxes %.1f ulps of their coordinate scale" % (name, worst["scores"], worst["boxes"]))
    assert worst["scores"] <= 4 and worst["boxes"] <= 4


# ---- NMS -----------------------------------------------------------------------------------------------------------
def run_nms(case, dev):
    c = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in case.items()}
    return K.det_nms(c["boxes"], c["scores"], c["groups"], c["valid"], c["thresh"], c["max_keep"], m_max=c["m_max"])


def check_nms(case, got):
    want = DC.oracle_nms(case)
    n = int(got["count"].item())
    assert n == want.numel()
    keep = got["keep"].cpu().long()
    assert torch.equal(keep[:n], want)
    assert bool((keep[n:] == -1).all())
    assert torch.equal(got["boxes"][:n].cpu(), case["boxes"][want])
    assert torch.equal(got["scores"][:n].cpu(), case["scores"][want])
    assert torch.equal(got["groups"][:n].cpu(), case["groups"][want])
    assert not got["boxes"][n:].any() and not got["scores"][n:].any() and not got["groups"][n:].any()


@pytest.mark.parametrize("name", list(DC.nms_cases()))
def test_nms(cuda, name):
    case = DC.nms_cases()[name]
    check_nms(case, run_nms(case, cuda))


def test_nms_reuses_workspace_across_sizes(cuda):
    """Calls with different n share the cached workspace: a large call, a small one, then the large one again."""
    C = DC.nms_cases()
    big, small = C["rpn_scale_0"], C["count_65"]
    check_nms(big, run_nms(big, cuda))
    check_nms(small, run_nms(small, cuda))
    check_nms(C["none_valid"], run_nms(C["none_valid"], cuda))
    check_nms(big, run_nms(big, cuda))


# ---- MultiScaleRoIAlign ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_size", [7, 14])
def test_roi_align(cuda, out_size):
    P = DC.roi_pyramid()
    boxes, count = DC.roi_boxes()
    r_max = boxes.shape[0]
    want, wlv = DC.oracle_roi_align(P, boxes, count, out_size)
    feats = [p[0].permute(1, 2, 0).unsqueeze(0).contiguous().to(cuda) for p in P]
    y = torch.full((r_max, out_size, out_size, DC.ROI_C), float("nan"), device=cuda)
    hi = torch.empty(y.shape, dtype=torch.float16, device=cuda)
    lo = torch.empty(y.shape, dtype=torch.float16, device=cuda)
    lv = torch.full((r_max,), -7, dtype=torch.int32, device=cuda)
    K.det_roi_align(feats, boxes.to(cuda), i32(count, cuda), out_size, levels=lv, y_f32=y, y_hi=hi, y_lo=lo)
    got_lv = lv[:count].cpu().long()
    bad = torch.where(got_lv != wlv)[0]
    assert bad.numel() == 0, "level differs from the oracle for boxes %s" % boxes[bad].tolist()
    assert bool((lv[count:] == -7).all())                    # levels past count are not written
    err = float((y.cpu() - want).abs().max())
    print("roi_align %d: max |gpu - oracle| %.3g (max |oracle| %.3g)" % (out_size, err, float(want.abs().max())))
    assert torch.equal(y.cpu(), want)                        # rows past count included: they are zero
    assert_operands(hi, lo, want, "roi_align")


# ---- box candidates --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(DC.box_candidate_cases()))
def test_box_candidates(cuda, name):
    case = DC.box_candidate_cases()[name]
    r_max = case["pred"].shape[0]
    ns = r_max * (DC.NC - 1)
    out = dict(boxes=torch.empty((ns, 4), device=cuda), scores=torch.empty(ns, device=cuda),
               groups=torch.empty(ns, dtype=torch.int32, device=cuda), valid=torch.empty(ns, dtype=torch.int32, device=cuda))
    K.det_box_candidates(case["pred"].to(cuda), DC.NC, case["props"].to(cuda), i32(case["count"], cuda), case["clip_hw"],
                         R.BOX_SCORE, R.BOX_MIN, D.XFORM_CLIP, out)
    wb, ws, wg, wv = DC.oracle_box_candidates(case)
    near = (ws - R.BOX_SCORE).abs() < 1e-6
    print("box_candidates %s: %d slots excluded from the valid comparison (score within 1e-6 of 0.05)" % (name, int(near.sum())))
    assert int(near.sum()) == 0
    assert torch.equal(out["valid"].cpu().bool(), wv)
    assert torch.equal(out["groups"].cpu().long(), wg)
    assert int(out["valid"].view(r_max, -1).sum(1).max()) <= 19            # m_max = 20 R in detectors.py
    raw = R.decode(case["pred"][:, DC.NC:DC.NC * 5], case["props"], (10.0, 10.0, 5.0, 5.0))[:, 1:].reshape(-1, 4)
    scale = torch.maximum(raw.abs().amax(1), ((raw[:, :2] + raw[:, 2:]) / 2).abs().amax(1))
    e_s, e_b = ulps(out["scores"], ws), box_ulps(out["boxes"], wb, scale)
    print("box_candidates %s: softmax %.1f ulps, boxes %.1f ulps of their coordinate scale" % (name, e_s, e_b))
    assert e_s <= 8 and e_b <= 4


# ---- mask probabilities, paste, person pick ----------------------------------------------------------------------------
def test_mask_probs(cuda):
    case = DC.mask_probs_case()
    d = case["raw"].shape[0]
    lg = torch.full((d, 28, 28), float("nan"), device=cuda)
    pr = torch.full((d, 28, 28), float("nan"), device=cuda)
    K.det_mask_probs(case["raw"].to(cuda), case["bias"].to(cuda), case["labels"].to(cuda), i32(case["count"], cuda), lg, pr)
    wl, wp = DC.oracle_mask_probs(case)
    assert torch.equal(lg.cpu(), wl)                       # labels 1 and 90; rows past count are zero
    e = ulps(pr, wp)
    print("mask_probs: sigmoid %.1f ulps" % e)
    assert e <= 4 and not pr[case["count"]:].any()


@pytest.mark.parametrize("name", list(DC.paste_cases()))
def test_paste_masks(cuda, name):
    case = DC.paste_cases()[name]
    d = case["boxes"].shape[0]
    H, W = case["to_hw"]
    masks = torch.full((d, 1, H, W), float("nan"), device=cuda)
    ob = torch.full((d, 4), float("nan"), device=cuda)
    K.det_paste_masks(case["probs"].to(cuda), case["boxes"].to(cuda), i32(case["count"], cuda), DC.paste_ratio(case), (H, W), masks, ob)
    wm, wb = DC.oracle_paste(case)
    assert torch.equal(ob.cpu(), wb)
    assert torch.equal(masks.cpu() != 0, wm != 0)          # the pasted region, truncated expanded corners included
    err = float((masks.cpu() - wm).abs().max())
    print("paste %s: max |gpu - oracle| %.3g" % (name, err))
    # inside the region the bilinear weights follow ATen's CPU kernel to within an ulp (its operation order is not
    # reproduced bit for bit): measured 1.19e-7 = one ulp below 1 on an H100
    assert err <= 2.0 ** -23


@pytest.mark.parametrize("ks", [0, 1, 3, 13])
@pytest.mark.parametrize("name", list(DC.person_cases()))
def test_person_mask(cuda, name, ks):
    case = DC.person_cases()[name]
    pid, box, m = K.det_person_mask(case["boxes"].to(cuda), case["labels"].int().to(cuda), i32(case["count"], cuda),
                                    case["masks"].to(cuda), 0.5, ks)
    wp, wb, wm = DC.oracle_person(case, ks)
    assert int(pid.item()) == wp
    assert torch.equal(box.cpu(), wb)
    assert torch.equal(m.cpu(), wm)


def test_person_mask_rejects_even_ks(cuda):
    case = DC.person_cases()["largest_negative_width"]
    with pytest.raises(LwbError, match="odd"):
        K.det_person_mask(case["boxes"].to(cuda), case["labels"].int().to(cuda), i32(6, cuda), case["masks"].to(cuda), 0.5, 4)


# ---- glue kernels --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(DC.TRANSFORM_HW))
def test_transform(cuda, name):
    img = DC.transform_cases()[name]
    ho, wo, hp, wp = DC.detector_sizes(*img.shape[1:])
    got = K.det_transform(img.to(cuda), ho, wo, hp, wp).cpu()
    want, hw = R.transform((img + 1) / 2.0)
    assert tuple(hw) == (ho, wo) and want.shape == got.shape
    err = float((got - want).abs().max())
    print("transform %s -> %dx%d: max |gpu - oracle| %.3g" % (name, ho, wo, err))
    # measured 0 on an H100 at every size: the per-pixel normalise and the bilinear blend round as ATen's CPU kernel does
    assert err == 0 and not got[..., ho:, :].any() and not got[..., wo:].any()


def test_stem_pool_odd_sizes_negative_windows(cuda):
    n, c, h, w = 2, 16, 37, 29
    x, scale, shift = DC.glue_tensors(11, (n, c, h, w), (c,), (c,))
    x[:, :4] = -(x[:, :4].abs() + 0.01)                      # channels whose every window is negative after the affine
    scale[:4], shift[:4] = 1.0, -0.5
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    hi = torch.empty((n, ho, wo, c), dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    K.det_stem_pool(x.to(cuda), scale.to(cuda), shift.to(cuda), hi, lo)
    want = F.max_pool2d(F.relu(x * scale[None, :, None, None] + shift[None, :, None, None]), 3, 2, 1).permute(0, 2, 3, 1)
    got = hi.cpu().float() + lo.cpu().float()
    err = float((got - want).abs().max() / want.abs().max())
    print("stem_pool: hi + lo vs oracle %.3g relative" % err)
    assert err <= 1e-6 and not hi[..., :4].any() and not lo[..., :4].any()


@pytest.mark.parametrize("variant", ["step2_raw2_ld", "res_half", "res_full"])
def test_bias_act(cuda, variant):
    n, c, ld = 2, 16, 24
    if variant == "step2_raw2_ld":
        h_in, w_in, h, w, step = 9, 8, 5, 4, 2
    else:
        h_in, w_in, h, w, step = 6, 10, 6, 10, 1
    raw, raw2, bias, res_f, res_h = DC.glue_tensors(12, (n, h_in, w_in, ld), (n, h_in, w_in, ld), (c,), (n, h, w, c),
                                                    (n, h // 2, w // 2, c))
    kw = dict(raw2=None, res=None, res_half=False, relu=True)
    v = raw[:, ::step, ::step, :c][:, :h, :w]
    if variant == "step2_raw2_ld":
        kw["raw2"] = raw2.to(cuda)
        v = v + raw2[:, ::step, ::step, :c][:, :h, :w]
    v = v + bias
    if variant == "res_half":
        kw.update(res=res_h.to(cuda), res_half=True)
        v = v + res_h.repeat_interleave(2, 1).repeat_interleave(2, 2)
    elif variant == "res_full":
        kw.update(res=res_f.to(cuda), relu=False)
        v = v + res_f
    if kw["relu"]:
        v = F.relu(v)
    y = torch.empty((n, h, w, c), device=cuda)
    hi = torch.empty(y.shape, dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    K.det_bias_act(raw.to(cuda), bias.to(cuda), step=step, out_hw=(h, w), c=c, y_f32=y, y_hi=hi, y_lo=lo, **kw)
    assert torch.equal(y.cpu(), v)
    assert_operands(hi, lo, v, "bias_act")


def test_d2s_bias_relu_is_conv_transpose(cuda):
    n, cin, c, h, w = 2, 8, 16, 5, 7
    x, wt, b = DC.glue_tensors(13, (n, cin, h, w), (cin, c, 2, 2), (c,))
    # the deconv as the engine runs it: a 1x1 conv to 4c columns, column (dy * 2 + dx) * c + co
    raw = torch.einsum("nihw,iokl->nhwklo", x.double(), wt.double()).reshape(n, h, w, 4 * c).float()
    y = torch.empty((n, 2 * h, 2 * w, c), device=cuda)
    hi = torch.empty(y.shape, dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    K.det_d2s_bias_relu(raw.to(cuda).contiguous(), b.to(cuda), y_f32=y, y_hi=hi, y_lo=lo)
    want = F.relu(F.conv_transpose2d(x.double(), wt.double(), b.double(), stride=2)).permute(0, 2, 3, 1)
    assert float((y.cpu().double() - want).abs().max()) <= 1e-6 * float(want.abs().max())
    exact = F.relu(raw.view(n, h, w, 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(n, 2 * h, 2 * w, c) + b)
    assert torch.equal(y.cpu(), exact)
    assert_operands(hi, lo, exact, "d2s")


# ---- end to end (synthetic weights) ----------------------------------------------------------------------------------
SEED = 21                               # tests/golden/maskrcnn.npz's weights


def detector(cuda, adjust=None):
    sd = S.synthetic_maskrcnn_state(SEED)
    if adjust:
        adjust(sd)
    det = D.PersonMaskRCNNDetector(ks=13, threshold=0.5, weights=sd)
    return det, sd


def test_zero_detections(cuda):
    def background(sd):
        sd["roi_heads.box_predictor.cls_score.bias"][0] += 30.0
    det, sd = detector(cuda, background)
    img = S.synthetic_source(256)[0]
    want, _ = R.forward((img + 1) / 2.0, D.remap_v1(sd))
    assert want["boxes"].shape[0] == 0
    out = det.forward([((img + 1) / 2.0).to(cuda)])[0]
    assert out["boxes"].shape == (0, 4) and out["labels"].numel() == 0 and out["scores"].numel() == 0
    assert out["masks"].shape == (0, 1, 256, 256)
    with pytest.raises(LwbError, match="nothing"):
        det.inference(img.to(cuda))
    # every buffer past the (zero) count holds zeros: no kernel used a stale row
    st = det.model.stream(256, 256)
    assert int(st.dets["count"].item()) == 0
    assert bool((st.dets["keep"] == -1).all())
    for t in (st.feats14.f32, st.mask_probs, st.mask_logits, st.masks, st.out_boxes, st.dets["boxes"], st.dets["scores"]):
        assert not t.any()


def test_no_person_takes_last_detection(cuda):
    def no_person(sd):
        sd["roi_heads.box_predictor.cls_score.bias"][1] -= 40.0
    det, sd = detector(cuda, no_person)
    img = S.synthetic_source(256)[0]
    want, _ = R.forward((img + 1) / 2.0, D.remap_v1(sd))
    assert want["boxes"].shape[0] > 0 and not bool((want["labels"] == 1).any())
    box, mask = det.inference(img.to(cuda))
    st = det.model.stream(256, 256)
    n = int(st.dets["count"].item())
    assert n == want["boxes"].shape[0] and not bool((st.dets["groups"][:n] == 1).any())
    assert torch.equal(box, st.out_boxes[n - 1])
    assert torch.equal(mask.cpu(), R.dilate((st.masks[n - 1:n].cpu() > 0.5).float(), 13))


def test_stream_reuse_leaks_no_state(cuda):
    det, _ = detector(cuda)
    m = det.model
    a, b = S.synthetic_source(256)[0].to(cuda), S.synthetic_source(256, seed=5)[0].to(cuda)

    def snap(img):
        st = m.run(img)
        torch.cuda.synchronize()
        n = int(st.dets["count"].item())
        return [t.clone() for t in (st.props["keep"], st.props["boxes"], st.dets["keep"], st.dets["boxes"], st.dets["scores"],
                                    st.mask_probs, st.masks, st.out_boxes, st.cand["boxes"], st.bcand["scores"])] + [n]

    first = snap(a)
    other = snap(b)
    again = snap(a)
    assert first[-1] > 0 and (other[-1] != first[-1] or not torch.equal(other[3], first[3]))
    for x, y in zip(first[:-1], again[:-1]):
        assert torch.equal(x, y)
    assert first[-1] == again[-1]
