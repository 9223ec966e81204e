"""The residency budget that lets the two sub-batch streams of ImpersonatorGenerator.inference overlap: the HBM-bound
kernels of one stream must fit on the SMs beside the other stream's persistent conv CTAs (DESIGN section 4, residency
budget).  A register or shared-memory increase in any of these kernels would silently serialise the streams again."""
import pytest
import torch

from impersonator_b200 import kernels as K
from impersonator_b200 import synthetic as S
from impersonator_b200.generator import ImpersonatorGenerator

pytestmark = pytest.mark.gpu

# blocks per SM beside one CTA of every conv instance the generator launches (DESIGN section 4)
CLAIMED_BESIDE = {"k_norm_act": 1, "k_norm_act<WARP> c=128": 1, "k_norm_act<WARP> c=256": 1, "k_norm_act<WARP> c=512": 1,
                  "k_heads": 2, "k_nchw_to_nhwc_split": 2}


def test_hbm_kernels_fit_beside_every_conv_instance(cuda):
    props = torch.cuda.get_device_properties(cuda)
    convs = {nm: K.conv_kernel_resources(*nm) for nm in K.GENERATOR_CONV_INSTANCES}
    for nm, c in convs.items():
        print("k_conv_wg<%d,%d>" % nm, c)
        assert c["local_bytes"] == 0, "conv instance %r spills" % (nm,)
        assert c["blocks_alone"] == 1 and c["threads"] == 384
    assert set(CLAIMED_BESIDE) == set(K.GENERATOR_GLUE_INSTANCES)
    for name, (which, ch) in K.GENERATOR_GLUE_INSTANCES.items():
        r = K.glue_kernel_resources(which, ch)
        beside = {nm: K.blocks_beside(c, r, props) for nm, c in convs.items()}
        print(name, r, beside)
        assert r["local_bytes"] == 0, "%s spills" % name
        for nm, b in beside.items():
            assert b >= CLAIMED_BESIDE[name], "%s: %d blocks beside k_conv_wg<%d,%d>" % (name, b, nm[0], nm[1])


def test_blocks_beside_matches_the_occupancy_api_without_a_conv(cuda):
    """With an empty 'conv' the arithmetic of blocks_beside is the occupancy calculator's own."""
    props = torch.cuda.get_device_properties(cuda)
    empty = dict(regs=0, threads=0, static_smem=0, dyn_smem=-1024)      # not even the 1 KB reserved per block
    for name, (which, ch) in K.GENERATOR_GLUE_INSTANCES.items():
        r = K.glue_kernel_resources(which, ch)
        assert K.blocks_beside(empty, r, props) == r["blocks_alone"], name


def test_two_streams_equal_one_stream_at_batch_16(cuda, monkeypatch):
    """The bench batch: two sub-batches of 8 (eager and as a captured graph) against one stream of 16."""
    from impersonator_b200.graph import CapturedStep
    torch.set_grad_enabled(False)
    n = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    n.load_state_dict(S.fill_state_dict(n.state_dict(), seed=0))
    n = n.to(cuda).eval()
    inp = S.synthetic_generator_inputs(16, 256, seed=35)
    enc, res = n.encode_src(inp["src"][:1].to(cuda))
    bg = (torch.rand(1, 3, 256, 256) * 2 - 1).to(cuda)
    tsf, T = inp["tsf"].to(cuda), inp["T"].to(cuda)
    monkeypatch.setenv("LWB_STREAMS", "1")
    one = [t.clone() for t in n.inference(enc, res, tsf, T, bg=bg)]
    monkeypatch.setenv("LWB_STREAMS", "2")
    two = [t.clone() for t in n.inference(enc, res, tsf, T, bg=bg)]
    step = CapturedStep(lambda tsf, T: n.inference(enc, res, tsf, T, bg=bg), dict(tsf=tsf, T=T))
    assert step.captured
    graph = step(tsf=tsf, T=T)
    torch.cuda.synchronize()
    assert any(k[0].startswith("inference#") for k in n.tsf_model._lwb_streams)
    d = max((a - b).abs().max().item() for a, b in zip(one, two))
    dg = max((a - b).abs().max().item() for a, b in zip(one, graph))
    print("batch 16: two streams vs one %.3e, captured %.3e" % (d, dg))
    assert d < 1e-5 and dg < 1e-5
