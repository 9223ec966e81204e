"""Every conv plan the networks bind (tests/conv_census.py: CENSUS), at its production descriptor and batch, in each operand
mode its network runs in, against the float64 emulation of that mode.

Per case: seeded N(0,1) operands built the way the networks build them (nchw_to_nhwc_split for fp16x3, the fp8 pair
blocks of norm_act_nhwc(lo_format=1) for fp16f8, the padded NHWC8 layout for the row-K stem), finite garbage in the input
channels between the layer's cin and cin_pad, weights at the layer's real shape packed with the arguments
PlanBinder.finalize uses.  ``out`` (NaN-filled) and ``stats`` sit between sentinel bands.  conv_census.check_output then
checks that every output element was written, that padded output channels are +0, the statistics against the output's
own sums, and windows of whole tiles against the emulation (EMU_BAR) and fp32 (FP32_BAR) with the padded input channels
zero in the reference: padded weight columns are zero, so garbage there cannot reach the result.  A second run into the
same buffers must give the same bytes: each output element is written by one tile, in a fixed order."""
import pytest
import torch

import conv_census as C
from conv_emulation import assert_bands_intact, guarded, to_f8_operands
from impersonator_b200 import kernels as K
from impersonator_b200._lib import ConvDesc
from impersonator_b200.binding import merge_transposed_weight

pytestmark = pytest.mark.gpu

CASES = [(e, s) for e in C.CENSUS for s in e.splits]


def operands(cuda, e, x, split):
    """The plan's (x, x1) operand pairs from the NCHW input x."""
    d = C.desc_of(e)
    if d["rowk"]:
        right = d["row_pitch"] - d["w_in"] - 3
        return K.nchw_to_nhwc_split(x.to(cuda), c_pad=8, pad_hw=(3, 3, 3, right), split=split), None
    parts = [x[:, :d["cin0"]], x[:, d["cin0"]:]] if d["cin1"] else [x]
    ops = [to_f8_operands(cuda, p) if split == 2 else K.nchw_to_nhwc_split(p.to(cuda), split=split) for p in parts]
    return ops[0], (ops[1] if d["cin1"] else None)


def pack(cuda, e, w, split):
    d = C.desc_of(e)
    absmax = float(w.abs().max())
    if d["rowk"]:
        return K.pack_conv_weight_rowk(w.to(cuda), cout_pad=e.cout_pad, cpx=e.cin_pad, split=split, absmax=absmax)
    wb = merge_transposed_weight(w.to(cuda)) if d["transposed"] == 2 else w.to(cuda)
    assert tuple(wb.shape) == e.weight
    return K.pack_conv_weight(wb, transposed=d["transposed"] == 1, cout_pad=e.cout_pad, cin_pad=e.cin_pad, split=split,
                              absmax=absmax)


@pytest.mark.parametrize("entry,split", CASES, ids=["%s-s%d" % (e.name, s) for e, s in CASES])
def test_census_plan(cuda, entry, split):
    e, d = entry, dict(C.desc_of(entry), split=split)
    name = C.label(e, split)
    x, w = C.make_inputs(e, seed=len(e.name))
    xs, x1s = operands(cuda, e, x, split)
    assert tuple(xs[0].shape) == e.x and (x1s is None or tuple(x1s[0].shape) == e.x1), name
    wp = pack(cuda, e, w, split)
    obuf, out = guarded(cuda, (d["n"], d["h_out"], d["w_out"], d["cout"]), torch.float32, float("nan"))
    sbuf, st = guarded(cuda, (d["n"], d["cout"], 2), torch.float64, 0.0) if e.stats else (None, None)
    plan = K.ConvPlan(ConvDesc(w_exp=15, **d), xs, x1s, wp, out, st)
    plan.run()
    torch.cuda.synchronize()
    assert_bands_intact(name + " out", obuf)
    if sbuf is not None:
        assert_bands_intact(name + " stats", sbuf)
    C.check_output(e, split, x, w, wp.w_exp, out, st.clone() if st is not None else None)
    first = out.clone()
    plan.run()                                   # once more into the same buffers: the same bytes
    torch.cuda.synchronize()
    same = first.view(torch.int32) == out.view(torch.int32)
    assert bool(same.all()), "%s: a second run changed %d output elements, the first at %s" % (
        name, int((~same).sum()), tuple(int(v) for v in (~same).nonzero()[0]))
    assert_bands_intact(name + " out (second run)", obuf)
