"""The row-K 7x7 stem over 9 to 24 input channels (16 or 24 padded channels per pixel: two or three K stages of 64 per
filter row) against the float64 emulation of its own arithmetic (conv_emulation.check_conv: the emulation of the operand
mode, plain fp32, and the InstanceNorm statistics against the sums of the kernel's own output).

Cases: cin 9, 14, 16, 18 and 24 (the generator input of the 'par' map is 14 channels, of 'binary' 18); batch 1 and 16;
outputs that end inside a pixel tile (the stem's 64-channel plans run 32 x 8-pixel tiles) and 512 x 512; both operand
modes the stem runs in (fp16 and fp16x3: the generator builds it with split = min(split, 1), so no fp8 lo).  The
8-channel plan keeps its kernel instance and K loop."""
import pytest
import torch
import torch.nn.functional as F

from impersonator_b200 import kernels as K
from impersonator_b200.generator import stem_cin_pad
from conv_emulation import check_conv
from test_conv_gpu import rnd

pytestmark = pytest.mark.gpu


def plan_stem(cuda, x, wt, split, halo=False):
    """The generator's stem plan for x [n, cin, h, w]: padded NHWC input of stem_cin_pad(cin) channels (3 px border
    top / left / bottom, 5 right), [ky][cout][kx * c_pad + c] weights.  -> (plan, out, stats, w_exp)."""
    n, cin, h, w = x.shape
    c_pad = stem_cin_pad(cin)
    xs = K.nchw_to_nhwc_split(x.to(cuda), c_pad=c_pad, pad_hw=(3, 3, 3, 5), split=split)
    ws = K.pack_conv_weight_rowk(wt.to(cuda), cpx=c_pad, split=split)
    d = K.make_conv_desc(n, h, w, c_pad, 64, 7, 7, stride=1, pad=3, split=split, rowk=True, row_pitch=w + 8, halo=halo)
    out = torch.full((n, h, w, 64), float("nan"), dtype=torch.float32, device=cuda)
    st = torch.zeros((n, 64, 2), dtype=torch.float64, device=cuda)
    return K.ConvPlan(d, xs, None, ws, out, st), out, st, ws.w_exp


def run_wide_stem(cuda, x, wt, split, halo=False):
    plan, out, st, e = plan_stem(cuda, x, wt, split, halo)
    plan.run()
    torch.cuda.synchronize()
    return K.nhwc_to_nchw(out).cpu(), st.cpu(), e, plan


def check_stem(name, cuda, n, cin, h, w, split, seed, halo=False):
    x = rnd(n, cin, h, w, seed=seed)
    wt = rnd(64, cin, 7, 7, seed=seed + 1, scale=0.05)
    got, st, e, plan = run_wide_stem(cuda, x, wt, split, halo)
    check_conv(name, split, got, x, wt, lambda a, b: F.conv2d(a, b, padding=3), e, st)
    return plan


@pytest.mark.parametrize("split", [1, 0])
@pytest.mark.parametrize("cin", [9, 14, 16, 18, 24])
def test_wide_stem_partial_tiles(cuda, cin, split):
    """37 x 45 outputs: the last 32-row tile holds 5 rows, the last 8-pixel column tile 5 columns."""
    plan = check_stem("stem%d_37x45" % cin, cuda, 2, cin, 37, 45, split, seed=10 + cin)
    info = plan.launch_info()
    assert info == dict(n_tile=64, mode=split, k_stages=stem_cin_pad(cin) // 8, taps=7), info


@pytest.mark.parametrize("split", [1, 0])
@pytest.mark.parametrize("cin", [14, 18])
def test_wide_stem_batch16(cuda, cin, split):
    check_stem("stem%d_b16_40x44" % cin, cuda, 16, cin, 40, 44, split, seed=40 + cin)


@pytest.mark.parametrize("split", [1, 0])
def test_wide_stem_512(cuda, split):
    check_stem("stem18_512", cuda, 1, 18, 512, 512, split, seed=70)


def test_wide_stem_halo_plan(cuda):
    """LWB_HALO builds the stem as a halo plan: checked as such, then run by the same kernel."""
    check_stem("stem14_halo", cuda, 2, 14, 33, 17, 1, seed=80, halo=True)


@pytest.mark.parametrize("split", [1, 0])
def test_eight_channel_stem_keeps_its_instance(cuda, split):
    """The 6-channel stem of the default uv_seg generator still pads to 8 channels and runs one K stage per filter row
    on the same (N tile 64, operand mode) instance as before."""
    plan = check_stem("stem6_37x45", cuda, 2, 6, 37, 45, split, seed=90)
    assert plan.desc.cin0 == 8
    assert plan.launch_info() == dict(n_tile=64, mode=split, k_stages=1, taps=7)
