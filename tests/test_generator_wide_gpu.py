"""The generator conditioned on the wide maps: ImpersonatorGenerator(src_dim = tsf_dim = 14) ('par') and 18 ('binary'),
whose 7x7 stems run the row-K plan over 16 / 24 padded channels.  Checked against
  * the slices the REFERENCE modules produced (tests/golden/generator_wide.npz), and
  * the full outputs of oracle/generator_ref.py on CPU,
at the 1e-3 max-abs bar, in the fp16f8 (default) and fp16x3 modes; plus a captured CUDA graph and the two sub-batch
streams.  As for the 6-channel generator, every pass on these inputs leaves the operand-range flag clear."""
import numpy as np
import pytest
import torch

import generator_wide_cases as W
from impersonator_b200 import synthetic as S
from oracle import generator_ref as G

pytestmark = pytest.mark.gpu
TOL = 1e-3
MODES = ["fp16f8", "fp16x3"]


@pytest.fixture(scope="module", params=W.WIDTHS, ids=lambda c: "cin%d" % c)
def wide(request, cuda):
    torch.set_grad_enabled(False)
    net, sd = W.weights(request.param)
    return request.param, net.to(cuda).eval(), sd, np.load(W.GOLD)


def close(name, got, gold, full=None):
    """got (device NCHW) against its golden slice and, when given, the oracle's full tensor."""
    e_g = float(np.abs(got - gold).max())
    print("%-28s vs reference golden %.3e" % (name, e_g))
    assert e_g < TOL, name
    if full is not None:
        e_o = (full[0].cpu() - full[1]).abs().max().item()
        print("%-28s vs oracle (full)    %.3e" % (name, e_o))
        assert e_o < TOL, name


@pytest.mark.parametrize("mode", MODES)
def test_encode_src_and_stem(cuda, wide, mode):
    cin, net, sd, g = wide
    net.set_precision(mode)
    src = W.cases(cin)["front"]["src"]
    enc, res = net.encode_src(src.to(cuda))
    st = net.src_model._stream(src.to(cuda), True, 'inference')
    assert st.cin_pad == (16 if cin == 14 else 24)
    raw = st.enc_layers[0][0].out.permute(0, 3, 1, 2)            # the stem's pre-norm output (nothing else has its shape)
    close("w%d %s stem raw" % (cin, mode), W.stem_slice(raw), g["w%d_stem_raw" % cin])
    e_m, r_m = G.encode_src(src, sd)
    for i in range(4):
        close("w%d %s enc%d" % (cin, mode, i), W.feat(enc[i]), g["w%d_enc%d" % (cin, i)], (enc[i], e_m[i]))
    close("w%d %s res5" % (cin, mode), W.feat(res[5]), g["w%d_res5" % cin], (res[5], r_m[5]))
    assert not (net.range_status() & 3)


@pytest.mark.parametrize("mode", MODES)
def test_infer_front(cuda, wide, mode):
    cin, net, sd, g = wide
    net.set_precision(mode)
    f = W.cases(cin)["front"]
    outs = net.infer_front(f["src"].to(cuda), f["tsf"].to(cuda), f["T"].to(cuda))
    ref = G.infer_front(f["src"], f["tsf"], f["T"], sd)
    for name, a, b in zip(("src_img", "src_mask", "tsf_img", "tsf_mask"), outs, ref):
        close("w%d %s front %s" % (cin, mode, name), W.sl(a), g["w%d_front_%s" % (cin, name)], (a, b))
    assert not (net.range_status() & 3)


@pytest.mark.parametrize("mode", MODES)
def test_inference(cuda, wide, mode):
    cin, net, sd, g = wide
    net.set_precision(mode)
    i2 = W.cases(cin)["inf"]
    enc, res = net.encode_src(i2["src"].to(cuda))
    img, mask = net.inference(enc, res, i2["tsf"].to(cuda), i2["T"].to(cuda))
    e_m, r_m = G.encode_src(i2["src"], sd)
    img_m, mask_m = G.inference(e_m, r_m, i2["tsf"], i2["T"], sd)
    close("w%d %s inference img" % (cin, mode), W.sl(img), g["w%d_inf_img" % cin], (img, img_m))
    close("w%d %s inference mask" % (cin, mode), W.sl(mask), g["w%d_inf_mask" % cin], (mask, mask_m))
    assert not (net.range_status() & 3)


@pytest.mark.parametrize("mode", MODES)
def test_swap(cuda, wide, mode):
    cin, net, sd, g = wide
    net.set_precision(mode)
    c = W.cases(cin)
    a, b = c["swap_a"], c["swap_b"]
    e12, r12 = net.encode_src(a["src"].to(cuda))
    e21, r21 = net.encode_src(b["src"].to(cuda))
    img, mask = net.swap(a["tsf"].to(cuda), e12, e21, r12, r21, a["T"].to(cuda), b["T"].to(cuda))
    o12, q12 = G.encode_src(a["src"], sd)
    o21, q21 = G.encode_src(b["src"], sd)
    m_img, m_mask = G.swap(a["tsf"], o12, o21, q12, q21, a["T"], b["T"], sd)
    close("w%d %s swap img" % (cin, mode), W.sl(img), g["w%d_swap_img" % cin], (img, m_img))
    close("w%d %s swap mask" % (cin, mode), W.sl(mask), g["w%d_swap_mask" % cin], (mask, m_mask))


def test_inference_512(cuda, wide):
    cin, net, sd, g = wide
    if cin != 18:
        pytest.skip("the 512 x 512 golden case is the 18-channel generator")
    net.set_precision(None)
    i5 = W.cases(cin)["inf512"]
    enc, res = net.encode_src(i5["src"].to(cuda))
    img, mask = net.inference(enc, res, i5["tsf"].to(cuda), i5["T"].to(cuda))
    close("w18 512 inference img", W.sl(img, 16), g["w18_512_inf_img"])
    close("w18 512 inference mask", W.sl(mask, 16), g["w18_512_inf_mask"])
    assert not (net.range_status() & 3)


def test_sub_batch_streams_and_graph_replay(cuda, wide, monkeypatch):
    """Batch 8 with shared source features: two sub-batch streams (LWB_STREAMS=2) against one stream and the oracle, then
    the same step captured as a CUDA graph and replayed."""
    from impersonator_b200.graph import CapturedStep
    cin, net, sd, _ = wide
    net.set_precision(None)
    inp = S.synthetic_generator_inputs(8, 256, seed=600 + cin, cin=cin)
    enc, res = net.encode_src(inp["src"].to(cuda))
    bg = (torch.rand(1, 3, 256, 256, generator=torch.Generator().manual_seed(cin)) * 2 - 1).to(cuda)
    tsf, T = inp["tsf"].to(cuda), inp["T"].to(cuda)
    monkeypatch.setenv("LWB_STREAMS", "1")
    c1, m1, p1 = [t.clone() for t in net.inference(enc, res, tsf, T, bg=bg)]
    monkeypatch.setenv("LWB_STREAMS", "2")
    c2, m2, p2 = [t.clone() for t in net.inference(enc, res, tsf, T, bg=bg)]
    assert any(k[0].startswith("inference#") for k in net.tsf_model._lwb_streams), "the sub-batch streams were not used"
    d = max((c1 - c2).abs().max().item(), (m1 - m2).abs().max().item(), (p1 - p2).abs().max().item())
    print("w%d two sub-batch streams vs one: %.3e" % (cin, d))
    assert d < 1e-5
    e_m, r_m = G.encode_src(inp["src"], sd)
    ref_c, ref_m = G.inference(e_m, r_m, inp["tsf"], inp["T"], sd)
    e = max((c2.cpu() - ref_c).abs().max().item(), (m2.cpu() - ref_m).abs().max().item())
    print("w%d two sub-batch streams vs oracle (full): %.3e" % (cin, e))
    assert e < TOL
    assert not (net.range_status() & 3)

    step = CapturedStep(lambda tsf, T: net.inference(enc, res, tsf, T, bg=bg), dict(tsf=tsf, T=T))
    assert step.captured
    other = S.synthetic_generator_inputs(8, 256, seed=700 + cin, cin=cin)
    want = [t.clone() for t in net.inference(enc, res, other["tsf"].to(cuda), other["T"].to(cuda), bg=bg)]
    got = step(tsf=other["tsf"].to(cuda), T=other["T"].to(cuda))
    torch.cuda.synchronize()
    d = max((a - b).abs().max().item() for a, b in zip(got, want))
    print("w%d graph replay vs eager: %.3e" % (cin, d))
    assert d < 1e-5

