"""GPU parity of the conv engine (wgmma implicit GEMM) and its glue kernels.  Every conv result is checked by
conv_emulation.check_conv: against a float64 emulation of its operand mode's own arithmetic (3e-5 of the output scale),
against plain torch fp32 on CPU (the same ATen ops the reference's nn.Conv2d / ConvTranspose2d call resolve to: 2e-4 for
fp16x3, 3e-4 for fp16f8, 2e-2 for single-pass fp16), and its InstanceNorm statistics against the sums of its own output."""
import pytest
import torch
import torch.nn.functional as F

from impersonator_b200 import kernels as K
from conv_emulation import check_conv, emulate_f8, report, to_f8_operands  # noqa: F401  (report, emulate_f8: used by the other conv tests)

pytestmark = pytest.mark.gpu


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def run_conv(cuda, x, w, stride=1, pad=1, dil=1, transposed=False, split=True, x1=None, n_tile=0, stats=True, halo=False,
             pad_w=None, out=None, st=None):
    """x [n,c,h,w] fp32 CPU, w OIHW (or IOHW when transposed) -> (NCHW fp32 CPU result, stats, the weights' w_exp).
    ``out`` / ``st``: caller-allocated NHWC output and statistics buffers (NaN- / zero-filled here otherwise)."""
    n, c0, h, wd = x.shape
    if int(split) == 2:
        xs, x1s = to_f8_operands(cuda, x), (to_f8_operands(cuda, x1) if x1 is not None else None)
    else:
        xs = K.nchw_to_nhwc_split(x.to(cuda), split=split)
        x1s = K.nchw_to_nhwc_split(x1.to(cuda), split=split) if x1 is not None else None
    ws = K.pack_conv_weight(w.to(cuda), transposed=transposed, split=split)
    cout = w.shape[1] if transposed else w.shape[0]
    kh, kw = w.shape[2:]
    d = K.make_conv_desc(n, h, wd, c0, cout, kh, kw, stride=stride, pad=pad, dil=dil,
                         cin1=0 if x1 is None else x1.shape[1], transposed=transposed, split=split, n_tile=n_tile,
                         halo=halo, pad_w=pad_w)
    if out is None:
        out = torch.full((n, d.h_out, d.w_out, cout), float("nan"), dtype=torch.float32, device=cuda)
    if st is None and stats:
        st = torch.zeros((n, cout, 2), dtype=torch.float64, device=cuda)
    plan = K.ConvPlan(d, xs, x1s, ws, out, st)
    plan.run()
    torch.cuda.synchronize()
    return K.nhwc_to_nchw(out).cpu(), (st.cpu() if st is not None else None), ws.w_exp


CASES = [
    # name, n, cin, cout, h, w, k, stride, pad, n_tile
    ("3x3_64_64_16x8", 1, 64, 64, 16, 8, 3, 1, 1, 0),
    ("3x3_64_64_32", 2, 64, 64, 32, 32, 3, 1, 1, 0),
    ("3x3_128_128_32", 2, 128, 128, 32, 32, 3, 1, 1, 0),
    ("3x3_512_512_32", 2, 512, 512, 32, 32, 3, 1, 1, 0),
    ("3x3_64_16_n16", 1, 64, 16, 32, 32, 3, 1, 1, 16),
    ("1x1_64_64", 1, 64, 64, 32, 32, 1, 1, 0, 0),
    ("3x3_s2_64_128_64", 2, 64, 128, 64, 64, 3, 2, 1, 0),
    ("3x3_s2_256_512_64", 1, 256, 512, 64, 64, 3, 2, 1, 0),
    ("3x3_ragged_40x24", 1, 64, 64, 40, 24, 3, 1, 1, 0),
    ("7x7_64_64", 1, 64, 64, 32, 32, 7, 1, 3, 0),
]


@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv2d(cuda, case, split):
    name, n, cin, cout, h, w, k, stride, pad, n_tile = case
    x = rnd(n, cin, h, w, seed=1)
    wt = rnd(cout, cin, k, k, seed=2, scale=0.05)
    got, st, e = run_conv(cuda, x, wt, stride=stride, pad=pad, split=split, n_tile=n_tile)
    check_conv(name, split, got, x, wt, lambda a, b: F.conv2d(a, b, stride=stride, padding=pad), e, st)


HALO_CASES = [c for c in CASES if c[7] == 1 and c[6] in (3, 7) and c[8] == c[6] // 2] + [
    ("7x7_64_16_heads", 2, 64, 16, 48, 40, 7, 1, 3, 16),
    ("5x5_64_64", 1, 64, 64, 32, 32, 5, 1, 2, 0),
    ("3x3_128_64_64x64", 2, 128, 64, 64, 64, 3, 1, 1, 0),
]


@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("case", HALO_CASES, ids=[c[0] for c in HALO_CASES])
def test_conv2d_halo(cuda, case, split):
    """Halo plans (lwb_conv_desc.halo = 1): accepted for stride-1 'same' convs and computed by the per-tap kernel, with the
    plain plan's accuracy."""
    name, n, cin, cout, h, w, k, stride, pad, n_tile = case
    x = rnd(n, cin, h, w, seed=31)
    wt = rnd(cout, cin, k, k, seed=32, scale=0.05)
    got, st, e = run_conv(cuda, x, wt, stride=1, pad=pad, split=split, n_tile=n_tile, halo=True)
    check_conv(name + "/halo", split, got, x, wt, lambda a, b: F.conv2d(a, b, padding=pad), e, st)


@pytest.mark.parametrize("split", [True, False])
def test_conv_concat_inputs_halo(cuda, split):
    a, b = rnd(2, 64, 32, 32, seed=5), rnd(2, 128, 32, 32, seed=6)
    wt = rnd(64, 192, 3, 3, seed=7, scale=0.05)
    got, st, e = run_conv(cuda, a, wt, split=split, x1=b, halo=True)
    check_conv("concat/halo", split, got, torch.cat([a, b], dim=1), wt, lambda xx, ww: F.conv2d(xx, ww, padding=1), e, st)


@pytest.mark.parametrize("split", [True, False])
def test_conv_transpose(cuda, split):
    conv = lambda a, b: F.conv_transpose2d(a, b, stride=2, padding=1, output_padding=1)      # noqa: E731
    for cin, cout, h in ((128, 64, 32), (512, 256, 32)):
        x = rnd(2, cin, h, h, seed=3)
        wt = rnd(cin, cout, 3, 3, seed=4, scale=0.05)
        got, st, e = run_conv(cuda, x, wt, stride=2, pad=1, transposed=True, split=split)
        check_conv("convT_%d_%d" % (cin, cout), split, got, x, wt, conv, e, st)


@pytest.mark.parametrize("split", [True, False])
def test_conv_concat_inputs(cuda, split):
    """skippers: conv(cat[skip, d]) without materialising the cat (networks/generator.py:177-179)."""
    a, b = rnd(2, 64, 32, 32, seed=5), rnd(2, 128, 32, 32, seed=6)
    wt = rnd(64, 192, 3, 3, seed=7, scale=0.05)
    got, st, e = run_conv(cuda, a, wt, split=split, x1=b)
    check_conv("concat", split, got, torch.cat([a, b], dim=1), wt, lambda xx, ww: F.conv2d(xx, ww, padding=1), e, st)


def run_stem(cuda, x, wt, split, halo=False):
    """The 7x7 stem (6 -> 64 channels) through the row-K layout: padded NHWC8 input, [ky][cout][kx*8 + c] weights."""
    n, _, h, w = x.shape
    xs = K.nchw_to_nhwc_split(x.to(cuda), c_pad=8, pad_hw=(3, 3, 3, 5), split=split)
    ws = K.pack_conv_weight_rowk(wt.to(cuda), split=split)
    d = K.make_conv_desc(n, h, w, 8, 64, 7, 7, stride=1, pad=3, split=split, rowk=True, row_pitch=w + 8, halo=halo)
    out = torch.full((n, h, w, 64), float("nan"), dtype=torch.float32, device=cuda)
    st = torch.zeros((n, 64, 2), dtype=torch.float64, device=cuda)
    K.ConvPlan(d, xs, None, ws, out, st).run()
    torch.cuda.synchronize()
    return K.nhwc_to_nchw(out).cpu(), st.cpu(), ws.w_exp


@pytest.mark.parametrize("halo", [False, True])
@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("size", [32, 256])
def test_stem_7x7_rowk(cuda, split, size, halo):
    """7x7 stem (6 -> 64 channels) through the row-K layout (networks/generator.py:80-84)."""
    x = rnd(2, 6, size, size, seed=8)
    wt = rnd(64, 6, 7, 7, seed=9, scale=0.05)
    got, st, e = run_stem(cuda, x, wt, split, halo=halo)
    check_conv("stem_rowk_%d" % size, split, got, x, wt, lambda a, b: F.conv2d(a, b, padding=3), e, st)


def test_heads_7x7(cuda):
    x = rnd(2, 64, 64, 96, seed=10)
    w_img, w_att = rnd(3, 64, 7, 7, seed=11, scale=0.02), rnd(1, 64, 7, 7, seed=12, scale=0.02)
    ref = F.conv2d(x, torch.cat([w_img, w_att]), padding=3)
    xn = x.permute(0, 2, 3, 1).contiguous().to(cuda)
    raw = K.conv7x7_heads_nhwc(xn, K.pack_head_weights(w_img.to(cuda), w_att.to(cuda)))
    got = raw.permute(0, 3, 1, 2).cpu()
    assert report("heads", got, ref) < 1e-5
    bg = rnd(1, 3, 64, 96, seed=13)
    color, mask, pred = K.heads_composite(raw, bg.to(cuda))
    rc, rm = torch.tanh(ref[:, :3]), torch.sigmoid(ref[:, 3:])
    assert (color.cpu() - rc).abs().max() < 1e-5 and (mask.cpu() - rm).abs().max() < 1e-5
    assert (pred.cpu() - (rm * bg + (1 - rm) * rc)).abs().max() < 1e-5       # models/imitator.py:331


def test_norm_act_warp(cuda):
    """IN + ReLU + residual + LWB warp-add (networks/generator.py:13-20,283-295,303-320)."""
    n, c, h, w = 3, 64, 32, 32
    raw = rnd(n, c, h, w, seed=14) * 2 + 0.5
    gamma, beta = 1 + 0.1 * rnd(c, seed=15), 0.1 * rnd(c, seed=16)
    res = rnd(n, c, h, w, seed=17)
    src = rnd(1, c, h, w, seed=18)
    from impersonator_b200 import synthetic as S
    T = S.synthetic_flow(n, 256, seed=3)
    for ac in (False, True):
        Ts = F.interpolate(T.permute(0, 3, 1, 2), size=(h, w), mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
        warp = F.grid_sample(src.expand(n, -1, -1, -1), Ts, mode="bilinear", padding_mode="zeros", align_corners=ac)
        ref = F.relu(F.instance_norm(raw, weight=gamma, bias=beta, eps=1e-5)) + res + warp
        nh = lambda t: t.permute(0, 2, 3, 1).contiguous().to(cuda)
        raw_d = nh(raw)
        st = K.instance_stats_nhwc(raw_d)
        y = torch.empty_like(raw_d)
        hi = torch.empty(raw_d.shape, dtype=torch.float16, device=cuda)
        lo = torch.empty_like(hi)
        ws = torch.empty((n, c, 2), dtype=torch.float32, device=cuda)
        K.norm_act_nhwc(raw_d, st, gamma.to(cuda), beta.to(cuda), True, ws, residual=nh(res), warp_src=nh(src),
                        T=T.to(cuda), align_corners=ac, y_f32=y, y_hi=hi, y_lo=lo)
        got = y.permute(0, 3, 1, 2).cpu()
        assert report("norm_act ac=%s" % ac, got, ref) < 2e-5
        rec = (hi.float() + lo.float()).permute(0, 3, 1, 2).cpu()
        assert (rec - got).abs().max() < 1e-5


@pytest.mark.parametrize("ac", [False, True])
def test_warp_nchw(cuda, ac):
    from impersonator_b200 import synthetic as S
    x = rnd(1, 24, 64, 64, seed=19)
    T = S.synthetic_flow(2, 256, seed=4)
    Ts = F.interpolate(T.permute(0, 3, 1, 2), size=(64, 64), mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    ref = F.grid_sample(x.expand(2, -1, -1, -1), Ts, mode="bilinear", padding_mode="zeros", align_corners=ac)
    got = K.warp_nchw(x.to(cuda), T.to(cuda), align_corners=ac).cpu()
    assert report("transform", got, ref) < 2e-5
    img = rnd(2, 3, 256, 256, seed=20)
    ref2 = F.grid_sample(img, T, mode="bilinear", padding_mode="zeros", align_corners=ac)
    got2 = K.warp_nchw(img.to(cuda), T.to(cuda), align_corners=ac).cpu()
    assert report("stn", got2, ref2) < 2e-5


def test_direct_conv(cuda):
    x = rnd(1, 5, 40, 40, seed=21)
    for (co, k, s, p, d) in ((8, 5, 1, 2, 1), (6, 4, 2, 1, 1), (7, 3, 1, 4, 4), (3, 1, 1, 0, 1)):
        wt, b = rnd(co, 5, k, k, seed=22, scale=0.1), rnd(co, seed=23)
        ref = F.conv2d(x, wt, b, stride=s, padding=p, dilation=d)
        got = K.conv2d_direct_nchw(x.to(cuda), wt.to(cuda), b.to(cuda), stride=s, pad=p, dil=d).cpu()
        assert report("direct k%d s%d d%d" % (k, s, d), got, ref) < 1e-5


F8_CASES = [c for c in CASES if c[2] % 64 == 0 and c[9] != 16]


@pytest.mark.parametrize("case", F8_CASES, ids=[c[0] for c in F8_CASES])
def test_conv2d_fp16f8(cuda, case):
    """split = 2: x_hi*w_hi on the fp16 path + (x*w_lo, x_lo*w) as e4m3 MMAs into the same accumulator."""
    name, n, cin, cout, h, w, k, stride, pad, n_tile = case
    x = rnd(n, cin, h, w, seed=1)
    wt = rnd(cout, cin, k, k, seed=2, scale=0.05)
    got, st, e = run_conv(cuda, x, wt, stride=stride, pad=pad, split=2, n_tile=n_tile)
    check_conv(name, 2, got, x, wt, lambda a, b: F.conv2d(a, b, stride=stride, padding=pad), e, st)


def test_conv_transposed_and_concat_fp16f8(cuda):
    x = rnd(2, 128, 32, 32, seed=5)
    wt = rnd(128, 64, 3, 3, seed=6, scale=0.05)
    got, _, e = run_conv(cuda, x, wt, stride=2, pad=1, transposed=True, split=2, stats=False)
    check_conv("convT 128->64", 2, got, x, wt, lambda a, b: F.conv_transpose2d(a, b, stride=2, padding=1, output_padding=1),
               e, emu_bar=1e-5)
    a, b = rnd(1, 64, 64, 64, seed=7), rnd(1, 64, 64, 64, seed=8)
    w2 = rnd(64, 128, 3, 3, seed=9, scale=0.05)
    got, st, e = run_conv(cuda, a, w2, split=2, x1=b)
    check_conv("concat 64+64->64", 2, got, torch.cat([a, b], dim=1), w2, lambda xx, ww: F.conv2d(xx, ww, padding=1), e, st)


@pytest.mark.parametrize("split", [1, 2])
def test_conv_homogeneity_and_batch_invariance_at_full_batch(cuda, split):
    """Size-independent properties at the BASELINE batch (16 x 512 x 32 x 32, the residual-block layer): conv(2x) = 2 conv(x)
    up to the fp16-subnormal rounding of the lo operands (|lo| < 6e-5 loses bits, so not bit-exact), and every image of a
    batch of identical images gets the same bits (same tile schedule, same accumulation order)."""
    x1 = rnd(1, 512, 32, 32, seed=3)
    x = x1.expand(16, -1, -1, -1).contiguous()
    wt = rnd(512, 512, 3, 3, seed=4, scale=0.02)
    y, _, _ = run_conv(cuda, x, wt, split=split, stats=False)
    y2, _, _ = run_conv(cuda, 2 * x, wt, split=split, stats=False)
    assert report("conv(2x) vs 2 conv(x)", y2, 2 * y) < 2e-5
    assert torch.equal(y[0], y[15]) and torch.equal(y[0], y[7])
    ref = F.conv2d(x1, wt, padding=1)
    assert report("512->512 @32 batch 16 (image 0)", y[:1], ref) < (2e-4 if split == 1 else 3e-4)


# Shapes the round-2 callers add: tiny images under one 16x8 tile (HMR layer3/4: 14x14, 7x7), 1x1 filters with up to 2048
# input channels, N tile 32 (folded heads, gated 16-channel layers, q/k/v), dilation 16, 5x5, 4x4 stride 2.
R2_CASES = [
    # name, n, cin, cout, h, w, k, stride, pad, dil, n_tile
    ("hmr_1x1_2048_512_7x7", 3, 2048, 512, 7, 7, 1, 1, 0, 1, 0),
    ("hmr_3x3_512_512_7x7", 3, 512, 512, 7, 7, 3, 1, 1, 1, 0),
    ("hmr_3x3_s2_256_256_14", 3, 256, 256, 14, 14, 3, 2, 1, 1, 0),
    ("hmr_1x1_64_256_56", 1, 64, 256, 56, 56, 1, 1, 0, 1, 0),
    ("hmr_3x3_s2_64_64_56", 2, 64, 64, 56, 56, 3, 2, 1, 1, 0),
    ("n32_3x3_64_32", 1, 64, 32, 40, 24, 3, 1, 1, 1, 0),
    ("attn_1x1_128_160", 1, 128, 160, 64, 64, 1, 1, 0, 1, 0),
    ("inp_3x3_dil16_128_256", 1, 128, 256, 64, 64, 3, 1, 16, 16, 0),
    ("inp_5x5_64_64", 1, 64, 64, 64, 64, 5, 1, 2, 1, 0),
    ("inp_4x4_s2_64_128", 1, 64, 128, 64, 64, 4, 2, 1, 1, 0),
]


@pytest.mark.parametrize("split", [1, 2])
@pytest.mark.parametrize("case", R2_CASES, ids=[c[0] for c in R2_CASES])
def test_conv2d_round2_shapes(cuda, case, split):
    name, n, cin, cout, h, w, k, stride, pad, dil, n_tile = case
    x = rnd(n, cin, h, w, seed=11)
    wt = rnd(cout, cin, k, k, seed=12, scale=0.05)
    got, st, e = run_conv(cuda, x, wt, stride=stride, pad=pad, dil=dil, split=split, n_tile=n_tile)
    check_conv(name, split, got, x, wt, lambda a, b: F.conv2d(a, b, stride=stride, padding=pad, dilation=dil), e, st)


@pytest.mark.parametrize("split", [1, 2])
def test_conv_7x1_folded_heads(cuda, split):
    """The 7x7 heads as a 7x1 filter with N = 7 columns x 4 channels (generator.fold_head_weights) + the column sum in
    lwb_heads_composite(folded_kw=7): the raw plan output against the emulation of the 7x1 conv, the composite against
    F.conv2d + tanh / sigmoid."""
    from impersonator_b200.generator import fold_head_weights
    n, h, w = 2, 48, 40
    x = rnd(n, 64, h, w, seed=21)
    w_img, w_att = rnd(3, 64, 7, 7, seed=22, scale=0.02), rnd(1, 64, 7, 7, seed=23, scale=0.02)
    folded = fold_head_weights(w_img, w_att)
    raw, _, e = run_conv(cuda, x, folded, stride=1, pad=3, pad_w=0, split=split, n_tile=32, stats=False)
    check_conv("folded 7x1 raw", split, raw, x, folded, lambda a, b: F.conv2d(a, b, padding=(3, 0)), e)
    raw_nhwc = raw.permute(0, 2, 3, 1).contiguous().to(cuda)
    color, mask, _ = K.heads_composite(raw_nhwc, None, folded_kw=7)
    ref_c = torch.tanh(F.conv2d(x, w_img, padding=3))
    ref_m = torch.sigmoid(F.conv2d(x, w_att, padding=3))
    d = max((color.cpu() - ref_c).abs().max().item(), (mask.cpu() - ref_m).abs().max().item())
    print("folded 7x1 heads split %d vs torch: %.3e" % (split, d))
    assert d < 2e-4


def run_merged_transposed(cuda, x, wt, split, out=None, st=None):
    """ConvTranspose2d(k3, s2, p1, op1) as one merged-phase plan (lwb_conv_desc.transposed = 2)."""
    from impersonator_b200.generator import merge_transposed_weight
    n, cin, h, w = x.shape
    cout = wt.shape[1]
    xs = to_f8_operands(cuda, x) if split == 2 else K.nchw_to_nhwc_split(x.to(cuda), split=split)
    ws = K.pack_conv_weight(merge_transposed_weight(wt.to(cuda)), split=split)
    d = K.make_conv_desc(n, h, w, cin, cout, 3, 3, stride=2, pad=1, transposed=True, split=split)
    d.transposed = 2
    if out is None:
        out = torch.full((n, 2 * h, 2 * w, cout), float("nan"), device=cuda)
    if st is None:
        st = torch.zeros(n, cout, 2, dtype=torch.float64, device=cuda)
    plan = K.ConvPlan(d, xs, None, ws, out, st)
    assert plan.num_launches == 1
    plan.run()
    torch.cuda.synchronize()
    return K.nhwc_to_nchw(out).cpu(), st.cpu(), ws.w_exp


@pytest.mark.parametrize("split", [1, 2, 0])
@pytest.mark.parametrize("cin,cout,h", [(128, 64, 32), (256, 128, 24)])
def test_conv_transposed_merged_phases(cuda, split, cin, cout, h):
    """lwb_conv_desc.transposed = 2: ConvTranspose2d(k3, s2, p1, op1) as ONE stride-1 pass with the four sub-pixel phases
    stacked on N (generator.merge_transposed_weight), against F.conv_transpose2d; statistics shared by the four phases."""
    x = rnd(2, cin, h, 40, seed=51)
    wt = rnd(cin, cout, 3, 3, seed=52, scale=0.05)
    got, st, e = run_merged_transposed(cuda, x, wt, split)
    check_conv("merged convT %d->%d" % (cin, cout), split, got, x, wt,
               lambda a, b: F.conv_transpose2d(a, b, stride=2, padding=1, output_padding=1), e, st)
