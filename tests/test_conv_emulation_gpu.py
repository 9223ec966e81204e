"""Conv-engine cases the layer tests cannot take as extra inputs, all checked against float64:

* output domains one pixel past a tile boundary (w % 8 == 1; h % 16 == 1 for the 16-row tiles, h % 32 == 1 for the
  32-row tiles of the swapped orientation), in all three operand modes;
* write-domain canaries: ``out`` and ``stats`` as views inside larger buffers whose sentinel bands must come back
  bit-identical;
* a weight-scale sweep: weights N(0,1) * s for s from 0.5 down to 3e-5 (fp16x3 against a float64 conv at 3e-5, fp16f8
  at its 3e-4 bar), which the per-layer weight exponent of the packers makes scale-independent;
* the operand formats the emulations assume, pinned bit for bit against torch restatements: fp16 is ``.half()`` (round
  to nearest even, subnormals included), e4m3 is ``clamp(+-448).to(torch.float8_e4m3fn)`` (what __NV_SATFINITE does), in
  the 64-channel pair-block layout of include/lwb_b200.h.
"""
import pytest
import torch
import torch.nn.functional as F

from impersonator_b200 import kernels as K
from conv_emulation import act_pair_blocks, assert_bands_intact, check_conv, fp16_pair, guarded, pair_blocks, report
from test_conv_gpu import rnd, run_conv, run_merged_transposed, run_stem

pytestmark = pytest.mark.gpu

SPLITS = [2, 1, 0]

# ---------------------------------------------------------------------------------------------------- tile boundaries
EDGE_CASES = [
    # name, n, cin, cout, h, w, n_tile
    ("n128_17x9", 2, 64, 128, 17, 9, 0),          # 16 x 8 tiles: one row and one column past the first tile
    ("n32_33x17", 2, 64, 32, 33, 17, 0),
    ("swapped_33x17", 2, 64, 64, 33, 17, 0),      # 32 x 8 tiles
    ("swapped_n64_65x25", 1, 64, 128, 65, 25, 64),
]


@pytest.mark.parametrize("split", SPLITS)
@pytest.mark.parametrize("case", EDGE_CASES, ids=[c[0] for c in EDGE_CASES])
def test_conv_one_past_tile_boundary(cuda, case, split):
    name, n, cin, cout, h, w, n_tile = case
    x = rnd(n, cin, h, w, seed=81)
    wt = rnd(cout, cin, 3, 3, seed=82, scale=0.05)
    got, st, e = run_conv(cuda, x, wt, pad=1, split=split, n_tile=n_tile)
    check_conv(name, split, got, x, wt, lambda a, b: F.conv2d(a, b, padding=1), e, st)


# ----------------------------------------------------------------------------------------------------------- canaries
CANARY_CASES = ["partial_plain", "swapped", "transposed_phases", "transposed_merged"]


@pytest.mark.parametrize("split", [1, 2])
@pytest.mark.parametrize("case", CANARY_CASES)
def test_conv_writes_only_its_domain(cuda, case, split):
    if case == "partial_plain":          # N = 128, 16 x 8 tiles, partial in y and x
        x, wt = rnd(2, 64, 20, 12, seed=83), rnd(128, 64, 3, 3, seed=84, scale=0.05)
        oshape, cout, conv = (2, 20, 12, 128), 128, lambda a, b: F.conv2d(a, b, padding=1)
    elif case == "swapped":              # N = 64, 32 x 8 tiles
        x, wt = rnd(2, 64, 40, 20, seed=85), rnd(64, 64, 3, 3, seed=86, scale=0.05)
        oshape, cout, conv = (2, 40, 20, 64), 64, lambda a, b: F.conv2d(a, b, padding=1)
    else:
        x = rnd(2, 128, 10, 6, seed=87)
        wt = rnd(128, 64, 3, 3, seed=88, scale=0.05)
        oshape, cout = (2, 20, 12, 64), 64
        conv = lambda a, b: F.conv_transpose2d(a, b, stride=2, padding=1, output_padding=1)      # noqa: E731
    obuf, out = guarded(cuda, oshape, torch.float32, float("nan"))
    sbuf, st = guarded(cuda, (2, cout, 2), torch.float64, 0.0)
    if case == "transposed_merged":
        got, stc, e = run_merged_transposed(cuda, x, wt, split, out=out, st=st)
    else:
        got, stc, e = run_conv(cuda, x, wt, stride=2 if case == "transposed_phases" else 1, pad=1,
                               transposed=case == "transposed_phases", split=split, out=out, st=st)
    assert_bands_intact(case + "/out", obuf)
    assert_bands_intact(case + "/stats", sbuf)
    check_conv(case, split, got, x, wt, conv, e, stc)


# ------------------------------------------------------------------------------------------------- weight-scale sweep
SCALES = [0.5, 0.05, 1e-3, 3e-4, 1e-4, 3e-5]
SWEEP_LAYERS = ["3x3_64_64_swapped", "3x3_128_128", "stem_7x7_rowk"]


@pytest.mark.parametrize("split", [1, 2])
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("layer", SWEEP_LAYERS)
def test_conv_weight_scale_sweep(cuda, layer, scale, split):
    """Accuracy must not depend on the weights' magnitude: unscaled fp16 packing puts w_lo of weights below ~1e-3 into
    the fp16 subnormals and loses up to 6e-4 (3x3, 64 -> 64, s = 3e-5) in fp16x3."""
    if layer == "stem_7x7_rowk" and split == 2:
        pytest.skip("the row-K stem has no fp16f8 path")
    if layer == "3x3_64_64_swapped":
        x, wt = rnd(1, 64, 24, 16, seed=91), rnd(64, 64, 3, 3, seed=92, scale=scale)
    elif layer == "3x3_128_128":
        x, wt = rnd(1, 128, 16, 16, seed=93), rnd(128, 128, 3, 3, seed=94, scale=scale)
    else:
        x, wt = rnd(1, 6, 40, 40, seed=95), rnd(64, 6, 7, 7, seed=96, scale=scale)
    pad = wt.shape[2] // 2
    conv = lambda a, b: F.conv2d(a, b, padding=pad)      # noqa: E731
    if layer == "stem_7x7_rowk":
        got, st, e = run_stem(cuda, x, wt, split)
    else:
        got, st, e = run_conv(cuda, x, wt, pad=pad, split=split)
    ref = conv(x.double(), wt.double())
    bar = 3e-5 if split == 1 else 3e-4
    assert report("%s s=%g split %d vs float64" % (layer, scale, split), got, ref) < bar
    check_conv("%s s=%g" % (layer, scale), split, got, x, wt, conv, e, st)


# ----------------------------------------------------------------------------------------------- operand formats
def special_values(shape, seed):
    """N(0,1) with a seventh of the entries replaced by each of: exact fp16 rounding ties, values whose residual is an
    fp16 subnormal (|v| ~ 1e-3), fp16-subnormal values themselves (~1e-6), values where e4m3(x_lo * 2^10) saturates
    (1024 <= |v| < 7168), values where e4m3(x / 16) saturates too (|v| >= 7168, including 7168 itself), and +-0."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(shape, generator=g).flatten()
    n = v.numel()
    kind = torch.randperm(n, generator=g) % 7
    h = (torch.randn(n, generator=g) * 4).half()
    nxt = (h.view(torch.int16) + 1).view(torch.float16)
    ties = (h.float() + nxt.float()) / 2                         # exactly halfway between two fp16 neighbours
    sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
    big = (1024 + torch.rand(n, generator=g) * 6000) * sign
    huge = (7168 + torch.rand(n, generator=g) * 20000) * sign
    huge[::5] = 7168.0 * sign[::5]
    big[::7] = 1024.0 * sign[::7]
    zeros = torch.where(sign > 0, 0.0, -0.0)
    for k, vals in ((1, ties), (2, torch.randn(n, generator=g) * 1e-3), (3, torch.randn(n, generator=g) * 1e-6),
                    (4, big), (5, huge), (6, zeros)):
        v = torch.where(kind == k, vals, v)
    return v.view(shape).float()


def assert_same_bits(name, got, want):
    g, w = got.cpu().contiguous().view(torch.uint8), want.contiguous().view(torch.uint8)
    assert g.shape == w.shape, (name, g.shape, w.shape)
    bad = (g != w).nonzero()
    assert bad.numel() == 0, "%s: %d bytes differ, first at %s (got %d, want %d)" % (
        name, bad.shape[0], tuple(bad[0].tolist()), int(g[tuple(bad[0])]), int(w[tuple(bad[0])]))


@pytest.mark.parametrize("split", [True, False])
def test_nchw_to_nhwc_split_bits(cuda, split):
    x = special_values((2, 20, 5, 7), seed=101)
    top, bottom, left, right = 1, 2, 3, 4
    hi, lo = K.nchw_to_nhwc_split(x.to(cuda), c_pad=32, pad_hw=(top, bottom, left, right), split=split)
    torch.cuda.synchronize()
    v = torch.zeros(2, 5 + top + bottom, 7 + left + right, 32)
    v[:, top:top + 5, left:left + 7, :20] = x.permute(0, 2, 3, 1)
    want_hi, want_lo = fp16_pair(v)
    assert_same_bits("nchw_to_nhwc hi", hi, want_hi)
    if split:
        assert_same_bits("nchw_to_nhwc lo", lo, want_lo)
    else:
        assert lo is None


@pytest.mark.parametrize("lo_format", [0, 1])
def test_norm_act_operand_bits(cuda, lo_format):
    """norm_act_nhwc without statistics or affine: y = raw, emitted as fp16 hi + (fp16 residual | fp8 pair blocks)."""
    raw = special_values((2, 5, 7, 128), seed=102)
    r = raw.to(cuda)
    y = torch.empty_like(r)
    hi = torch.empty(r.shape, dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    K.norm_act_nhwc(r, None, None, None, False, None, y_f32=y, y_hi=hi, y_lo=lo, lo_format=lo_format)
    torch.cuda.synchronize()
    assert_same_bits("norm_act y_f32", y, raw)
    want_hi, want_lo = fp16_pair(raw)
    assert_same_bits("norm_act hi", hi, want_hi)
    if lo_format == 0:
        assert_same_bits("norm_act lo", lo, want_lo)
    else:
        assert_same_bits("norm_act lo8", lo.view(torch.uint8), act_pair_blocks(raw, want_hi))


def test_gated_act_operand_bits(cuda):
    """gated_act_nhwc, lo_format 1, 100 channels padded to 128: the operands restated from its own fp32 output."""
    n, h, w, c, c_pad = 2, 5, 7, 100, 128
    a = special_values((n, h, w, c), seed=103)
    raw = torch.cat([a, torch.full((n, h, w, c), 100.0)], dim=-1).to(cuda)       # gate sigmoid(100) = 1
    y = torch.empty((n, h, w, c), device=cuda)
    hi = torch.empty((n, h, w, c_pad), dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    K.gated_act_nhwc(raw, c, None, 0, None, None, y_f32=y, y_hi=hi, y_lo=lo, lo_format=1)
    torch.cuda.synchronize()
    v = torch.zeros(n, h, w, c_pad)
    v[..., :c] = y.cpu()
    want_hi, _ = fp16_pair(v)
    assert_same_bits("gated hi", hi, want_hi)
    assert_same_bits("gated lo8", lo.view(torch.uint8), act_pair_blocks(v, want_hi))


def weights(kind, shape, seed):
    if kind == "special":
        return special_values(shape, seed)
    if kind == "small":                  # E = 26: scaled residuals are normal fp16, unscaled ones would be subnormal
        return rnd(*shape, seed=seed, scale=1e-4)
    return torch.zeros(shape)            # all-zero layer: E = 15


@pytest.mark.parametrize("kind", ["special", "small", "zero"])
@pytest.mark.parametrize("transposed", [False, True])
@pytest.mark.parametrize("split", [0, 1, 2])
def test_pack_conv_weight_bits(cuda, split, transposed, kind):
    cout, cin, cout_pad, cin_pad = 20, 40, 32, 64
    w = weights(kind, (cin, cout, 3, 3) if transposed else (cout, cin, 3, 3), seed=104)
    pw = K.pack_conv_weight(w.to(cuda), transposed=transposed, cout_pad=cout_pad, cin_pad=cin_pad, split=split)
    torch.cuda.synchronize()
    E = K.weight_exponent(w.abs().max())
    assert pw.w_exp == E and (kind != "zero" or E == 15)
    oihw = w.permute(1, 0, 2, 3) if transposed else w
    taps = torch.zeros(9, cout_pad, cin_pad)
    taps[:, :cout, :cin] = oihw.permute(2, 3, 0, 1).reshape(9, cout, cin)
    if split == 2:
        h = taps.half()
        assert_same_bits("pack f8 hi", pw[0], (h.float() * 2.0 ** E).half())
        assert_same_bits("pack f8 lo8", pw[1].view(torch.uint8),
                         pair_blocks((taps - h.float()) * 2.0 ** (E + 4), taps * 2.0 ** (E - 10)))
    else:
        want_hi, want_lo = fp16_pair(taps * 2.0 ** E)
        assert_same_bits("pack hi", pw[0], want_hi)
        if split:
            assert_same_bits("pack lo", pw[1], want_lo)
        else:
            assert pw[1] is None


@pytest.mark.parametrize("kind", ["special", "small", "zero"])
def test_pack_conv_weight_rowk_bits(cuda, kind):
    cout, cout_pad = 20, 32
    w = weights(kind, (cout, 6, 7, 7), seed=105)
    pw = K.pack_conv_weight_rowk(w.to(cuda), cout_pad=cout_pad, split=True)
    torch.cuda.synchronize()
    E = K.weight_exponent(w.abs().max())
    assert pw.w_exp == E
    full = torch.zeros(7, cout_pad, 8, 8)                        # [ky][co][kx][c], K index = kx * 8 + c
    full[:, :cout, :7, :6] = w.permute(2, 0, 3, 1)
    want_hi, want_lo = fp16_pair(full.reshape(7, cout_pad, 64) * 2.0 ** E)
    assert_same_bits("rowk hi", pw[0], want_hi)
    assert_same_bits("rowk lo", pw[1], want_lo)
